// chd_build.cuh — spatial-hash build: GetChannelId per entity (spatial.go:161-180) and a STABLE LSD radix
// sort of entity indices by cell (<= 2 passes of <= 10-bit digits: the spatial id space has < 2^19 cells,
// settings.go:94-95), then cell boundaries.  Result: cell_start[C+2], sorted_entity[N] ordered (cell asc,
// entity index asc) — the canonical order of SURVEY.md §8c'.  Invalid (out-of-world) entities get key C and
// sort to the tail [cell_start[C], cell_start[C+1]).
//
// Work decomposition: a fixed grid (multiple of the SM count); each block owns a CONTIGUOUS slice of the
// input processed in order, so global histograms are bins x nblocks (small) and stability is preserved.
// HBM traffic per pass: read key(+val) / write key+val, coalesced reads; per entity 16 B of positions are
// read once in the assign kernel.
#pragma once
#include "chd_types.cuh"

namespace chd {


// Block-aggregated append of the entities whose cell changed (the prefix of Notify, spatial.go:612-626): one global atomic per
// block and call, which every thread of the block makes.  Entity i moved from key p to key c; the list holds channel ids, 0 =
// outside the world (GetChannelId error, spatial.go:613-622).  reset: zero the block's counter for the next call.
__device__ __forceinline__ void handover_append(const GridDev& g, const HandoverOut& ho, uint32_t& s_cnt, uint32_t& s_base, bool moved,
                                                uint32_t i, uint32_t p, uint32_t c, bool reset) {
    uint32_t my = 0;
    if (moved) my = atomicAdd(&s_cnt, 1u);
    __syncthreads();
    if (threadIdx.x == 0) {
        if (s_cnt) s_base = atomicAdd(ho.count, s_cnt);
        if (reset) s_cnt = 0;
    }
    __syncthreads();
    if (moved) {
        const uint32_t slot = s_base + my;
        if (slot < ho.cap) {
            ho.entity[slot] = i;
            ho.src_cell[slot] = p >= g.cells ? 0u : p + g.id_start;
            ho.dst_cell[slot] = c >= g.cells ? 0u : c + g.id_start;
        }
    }
}

// A block's digit histogram in shared memory: cleared, then (after a barrier) written to column blockIdx.x of hist[digit][block]
template <int BINS>
__device__ __forceinline__ void hist_clear(uint32_t* s_hist) {
    for (int d = threadIdx.x; d < BINS; d += BUILD_THREADS) s_hist[d] = 0;
}
template <int BINS>
__device__ __forceinline__ void hist_flush(const uint32_t* s_hist, uint32_t* __restrict__ hist, uint32_t nblocks) {
    __syncthreads();
    for (int d = threadIdx.x; d < BINS; d += BUILD_THREADS) hist[(uint32_t)d * nblocks + blockIdx.x] = s_hist[d];
}

// Digit d's scanned base in block `block`'s column of hist_scanned.  Block 0's bases are the global exclusive counts per digit, so
// in a single-pass sort (digit == key) they are the cell CSR offsets: with ex.cell_start set, block 0 publishes them (keys ==
// cells mark out-of-world entities, so cell_start[cells] is the in-world count).  cell_start[cells + 1] = n is the caller's.
__device__ __forceinline__ uint32_t load_base(const uint32_t* __restrict__ hist_scanned, uint32_t d, uint32_t nblocks, uint32_t block,
                                              const ScatterExtras& ex) {
    const uint32_t b = hist_scanned[d * nblocks + block];
    if (ex.cell_start && block == 0) {
        if (d <= ex.cells) ex.cell_start[d] = b;
        if (d == ex.cells) *ex.n_in_world = b;
    }
    return b;
}

// A scatter block's bases (load_base of every digit) into s_base, and block 0 publishes the end of the cell CSR.
template <int BINS>
__device__ __forceinline__ void load_bases(uint32_t* s_base, const uint32_t* __restrict__ hist_scanned, uint32_t nblocks, uint32_t n,
                                           const ScatterExtras& ex) {
    for (int d = threadIdx.x; d < BINS; d += BUILD_THREADS) s_base[d] = load_base(hist_scanned, d, nblocks, blockIdx.x, ex);
    if (ex.cell_start && blockIdx.x == 0 && threadIdx.x == 0) ex.cell_start[ex.cells + 1] = n;
}

// Loads a tile's keys and values (warp w: the run of 32 * BUILD_ROUNDS from tile + w * 32 * BUILD_ROUNDS, one element per lane and
// round; val_in == nullptr: value = index) and ranks each element among the warp's earlier ones with the same digit: rk = the
// warp's count of the digit so far (wcnt, the warp's row of counters, which the lowest lane holding the digit advances) + the
// lane's rank among its peers.  Lanes past hi take part in the match only.
template <typename Cnt>
__device__ __forceinline__ void load_and_rank(const uint32_t* __restrict__ key_in, const uint32_t* __restrict__ val_in, uint32_t tile, uint32_t hi,
                                              uint32_t shift, uint32_t mask, Cnt* wcnt, uint32_t (&k)[BUILD_ROUNDS], uint32_t (&v)[BUILD_ROUNDS],
                                              uint32_t (&rk)[BUILD_ROUNDS]) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const uint32_t lt_mask = (1u << lane) - 1u;
#pragma unroll
    for (int r = 0; r < BUILD_ROUNDS; r++) {
        const uint32_t i = tile + w * (32 * BUILD_ROUNDS) + r * 32 + lane;
        const bool valid = i < hi;
        k[r] = valid ? key_in[i] : 0u;
        v[r] = valid ? (val_in ? val_in[i] : i) : 0u;
        const uint32_t d = valid ? ((k[r] >> shift) & mask) : 0xFFFFFFFFu;
        const uint32_t peers = __match_any_sync(0xffffffffu, d);
        const uint32_t rank = __popc(peers & lt_mask);
        uint32_t cnt = 0;
        if (valid) cnt = wcnt[d];
        __syncwarp();
        if (valid && rank == 0) wcnt[d] = (Cnt)(cnt + __popc(peers));
        __syncwarp();
        rk[r] = cnt + rank;
    }
}

// cell key per entity (+ optional handover detection against the previous build's keys:
// the prefix of Notify, spatial.go:612-626: GetChannelId(old) != GetChannelId(new)).
__global__ void __launch_bounds__(256) assign_cells_kernel(GridDev g, const double* __restrict__ x, const double* __restrict__ z,
                                                           uint32_t n, uint32_t* __restrict__ key,
                                                           const uint32_t* __restrict__ prev_key, HandoverOut ho,
                                                           unsigned long long* bump_epoch) {
    __shared__ uint32_t s_cnt, s_base;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (bump_epoch && i == 0) *bump_epoch = chd_next_epoch(*bump_epoch);  // (the border export's compaction follows in the same graph)
    if (prev_key) {
        if (threadIdx.x == 0) s_cnt = 0;
        __syncthreads();
    }
    uint32_t c = g.cells, p = g.cells;
    bool moved = false;
    if (i < n) {
        c = cell_index(g, x[i], z[i]);
        if (c == CHD_INVALID_CELL) c = g.cells;
        key[i] = c;
        if (prev_key) {
            p = prev_key[i];
            moved = p != c;
        }
    }
    if (prev_key) handover_append(g, ho, s_cnt, s_base, moved, i, p, c, false);
}

// assign_cells_kernel + the first pass's radix_hist_kernel in ONE launch (single-GPU build: one launch and one pass over the keys
// less on the critical path of a tick).  Same block decomposition as radix_hist_kernel: block b owns the contiguous slice
// [b * per_block, (b + 1) * per_block); handover candidates are appended with one global atomic per 256-entity step.
template <int BINS>
__global__ void __launch_bounds__(BUILD_THREADS)
    assign_hist_kernel(GridDev g, const double* __restrict__ x, const double* __restrict__ z, uint32_t n, uint32_t* __restrict__ key,
                       const uint32_t* __restrict__ prev_key, HandoverOut ho, uint32_t per_block, uint32_t mask, uint32_t* __restrict__ hist,
                       uint32_t nblocks, unsigned long long* bump_epoch) {
    __shared__ uint32_t s_hist[BINS];
    __shared__ uint32_t s_cnt, s_base;
    if (bump_epoch && blockIdx.x == 0 && threadIdx.x == 0) *bump_epoch = chd_next_epoch(*bump_epoch);
    hist_clear<BINS>(s_hist);
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    const uint32_t lo = min(n, blockIdx.x * per_block);
    const uint32_t hi = min(n, lo + per_block);
    for (uint32_t base = lo; base < hi; base += BUILD_THREADS) {
        const uint32_t i = base + threadIdx.x;
        uint32_t c = g.cells, p = g.cells;
        bool moved = false;
        if (i < hi) {
            c = cell_index(g, x[i], z[i]);
            if (c == CHD_INVALID_CELL) c = g.cells;
            key[i] = c;
            atomicAdd(&s_hist[c & mask], 1u);
            if (prev_key) {
                p = prev_key[i];
                moved = p != c;
            }
        }
        if (prev_key) {
            handover_append(g, ho, s_cnt, s_base, moved, i, p, c, true);
            __syncthreads();  // s_base is rewritten in the next step
        }
    }
    hist_flush<BINS>(s_hist, hist, nblocks);
}

// per-block digit histogram; hist layout [digit][block]
template <int BINS>
__global__ void __launch_bounds__(BUILD_THREADS)
    radix_hist_kernel(const uint32_t* __restrict__ key, uint32_t n, const uint32_t* __restrict__ n_ptr, uint32_t per_block,
                      uint32_t shift, uint32_t mask, uint32_t* __restrict__ hist, uint32_t nblocks, unsigned long long* bump_epoch) {
    __shared__ uint32_t s_hist[BINS];
    // first kernel of the build stage: opens a new epoch for the stage's look-back scans (chd_scan.cuh)
    if (bump_epoch && blockIdx.x == 0 && threadIdx.x == 0) *bump_epoch = chd_next_epoch(*bump_epoch);
    if (n_ptr) n = min(n, *n_ptr);  // live length on the device (multi-GPU: own + halo entities)
    hist_clear<BINS>(s_hist);
    __syncthreads();
    const uint32_t lo = min(n, blockIdx.x * per_block);
    const uint32_t hi = min(n, lo + per_block);
    for (uint32_t i = lo + threadIdx.x; i < hi; i += BUILD_THREADS) atomicAdd(&s_hist[(key[i] >> shift) & mask], 1u);
    hist_flush<BINS>(s_hist, hist, nblocks);
}

// stable scatter of one pass.  val_in == nullptr means "value = index" (first pass).
template <int BINS>
__global__ void __launch_bounds__(BUILD_THREADS)
    radix_scatter_kernel(const uint32_t* __restrict__ key_in, const uint32_t* __restrict__ val_in, uint32_t n,
                         const uint32_t* __restrict__ n_ptr, uint32_t per_block, uint32_t shift, uint32_t mask, const uint32_t* __restrict__ hist_scanned,
                         uint32_t nblocks, uint32_t* __restrict__ key_out, uint32_t* val_out, ScatterExtras ex) {
    __shared__ uint32_t s_base[BINS];
    __shared__ uint32_t s_tot[BINS];
    __shared__ uint32_t s_wcnt[BUILD_WARPS][BINS];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (n_ptr) n = min(n, *n_ptr);
    load_bases<BINS>(s_base, hist_scanned, nblocks, n, ex);
    const uint32_t lo = min(n, blockIdx.x * per_block);
    const uint32_t hi = min(n, lo + per_block);
    for (uint32_t tile = lo; tile < hi; tile += BUILD_TILE) {
        for (int d = threadIdx.x; d < BINS * BUILD_WARPS; d += BUILD_THREADS) (&s_wcnt[0][0])[d] = 0;
        __syncthreads();
        uint32_t k[BUILD_ROUNDS], v[BUILD_ROUNDS], rk[BUILD_ROUNDS];
        load_and_rank(key_in, val_in, tile, hi, shift, mask, s_wcnt[w], k, v, rk);
        __syncthreads();
        for (int d = threadIdx.x; d < BINS; d += BUILD_THREADS) {
            uint32_t run = 0;
#pragma unroll
            for (int ww = 0; ww < BUILD_WARPS; ww++) {
                const uint32_t c = s_wcnt[ww][d];
                s_wcnt[ww][d] = run;
                run += c;
            }
            s_tot[d] = run;
        }
        __syncthreads();
#pragma unroll
        for (int r = 0; r < BUILD_ROUNDS; r++) {
            const uint32_t i = tile + w * (32 * BUILD_ROUNDS) + r * 32 + lane;
            if (i < hi) {
                const uint32_t d = (k[r] >> shift) & mask;
                const uint32_t dst = s_base[d] + s_wcnt[w][d] + rk[r];
                val_out[dst] = v[r];
                if (key_out) key_out[dst] = k[r];
            }
        }
        __syncthreads();
        for (int d = threadIdx.x; d < BINS; d += BUILD_THREADS) s_base[d] += s_tot[d];
        __syncthreads();
    }
}

// The same pass for the bandwidth-bound regime (N >> 1 M): the tile is first reordered by digit in SHARED memory, then written
// out in sorted order, so consecutive threads store to consecutive addresses of a digit's run (full 32-byte sectors instead of
// one 4-byte store per sector: the plain scatter above writes 8x the DRAM sectors it needs at 65 536 cells).  Stable, same result.
template <int BINS>
__global__ void __launch_bounds__(BUILD_THREADS)
    radix_scatter_sorted_kernel(const uint32_t* __restrict__ key_in, const uint32_t* __restrict__ val_in, uint32_t n,
                                const uint32_t* __restrict__ n_ptr, uint32_t per_block, uint32_t shift, uint32_t mask,
                                const uint32_t* __restrict__ hist_scanned, uint32_t nblocks, uint32_t* __restrict__ key_out, uint32_t* val_out,
                                ScatterExtras ex) {
    __shared__ uint32_t s_base[BINS];   // global position of the next element of each digit
    __shared__ uint32_t s_lofs[BINS];   // exclusive prefix of the tile's digit counts = local position of each digit's run
    __shared__ uint16_t s_wcnt[BUILD_WARPS][BINS];
    __shared__ uint32_t s_key[BUILD_TILE], s_val[BUILD_TILE];
    __shared__ uint32_t s_scan[BUILD_WARPS];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    constexpr int DPT = BINS / BUILD_THREADS;  // digits per thread in the prefix step
    if (n_ptr) n = min(n, *n_ptr);
    load_bases<BINS>(s_base, hist_scanned, nblocks, n, ex);
    const uint32_t lo = min(n, blockIdx.x * per_block);
    const uint32_t hi = min(n, lo + per_block);
    for (uint32_t tile = lo; tile < hi; tile += BUILD_TILE) {
        for (int d = threadIdx.x; d < BINS * BUILD_WARPS; d += BUILD_THREADS) (&s_wcnt[0][0])[d] = 0;
        __syncthreads();
        uint32_t k[BUILD_ROUNDS], v[BUILD_ROUNDS], rk[BUILD_ROUNDS];
        load_and_rank(key_in, val_in, tile, hi, shift, mask, s_wcnt[w], k, v, rk);
        __syncthreads();
        // per digit: warp counts -> exclusive offsets across warps; tile totals -> exclusive prefix across digits
        uint32_t tot[DPT], sum = 0;
#pragma unroll
        for (int q = 0; q < DPT; q++) {
            const int d = threadIdx.x * DPT + q;
            uint32_t run = 0;
#pragma unroll
            for (int ww = 0; ww < BUILD_WARPS; ww++) {
                const uint32_t c = s_wcnt[ww][d];
                s_wcnt[ww][d] = (uint16_t)run;
                run += c;
            }
            tot[q] = run;
            sum += run;
        }
        uint32_t incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) s_scan[w] = incl;
        __syncthreads();
        uint32_t pre = incl - sum;
        for (int ww = 0; ww < w; ww++) pre += s_scan[ww];
#pragma unroll
        for (int q = 0; q < DPT; q++) {
            s_lofs[threadIdx.x * DPT + q] = pre;
            pre += tot[q];
        }
        __syncthreads();
        const uint32_t count = min((uint32_t)BUILD_TILE, hi - tile);
#pragma unroll
        for (int r = 0; r < BUILD_ROUNDS; r++) {
            const uint32_t i = tile + w * (32 * BUILD_ROUNDS) + r * 32 + lane;
            if (i < hi) {
                const uint32_t d = (k[r] >> shift) & mask;
                const uint32_t lp = s_lofs[d] + s_wcnt[w][d] + rk[r];
                s_key[lp] = k[r];
                s_val[lp] = v[r];
            }
        }
        __syncthreads();
        for (uint32_t j = threadIdx.x; j < count; j += BUILD_THREADS) {
            const uint32_t kk = s_key[j], d = (kk >> shift) & mask;
            const uint32_t dst = s_base[d] + (j - s_lofs[d]);
            val_out[dst] = s_val[j];
            if (key_out) key_out[dst] = kk;
        }
        __syncthreads();
        // advance the global bases by the tile's digit totals (= next digit's local offset - this digit's)
#pragma unroll
        for (int q = 0; q < DPT; q++) {
            const int d = threadIdx.x * DPT + q;
            s_base[d] += tot[q];
        }
        __syncthreads();
    }
}

// single-pass builds: the cell CSR offsets straight from the scanned histogram (load_base of block 0), published BEFORE the
// scatter runs so that the emit preparation can overlap it
__global__ void __launch_bounds__(256) publish_cell_start_kernel(const uint32_t* __restrict__ hist_scanned, uint32_t nblocks, uint32_t n,
                                                                 const uint32_t* __restrict__ n_ptr, ScatterExtras ex) {
    const uint32_t d = blockIdx.x * blockDim.x + threadIdx.x;
    if (n_ptr) n = min(n, *n_ptr);
    if (d <= ex.cells) load_base(hist_scanned, d, nblocks, 0, ex);
    if (d == 0) ex.cell_start[ex.cells + 1] = n;
}

// cell_start[c] = first sorted position whose key >= c, for c in [0, C+1]; cell_start[C+1] = n.
__global__ void __launch_bounds__(256)
    cell_bounds_kernel(const uint32_t* __restrict__ sorted_key, uint32_t n, const uint32_t* __restrict__ n_ptr, uint32_t cells,
                       uint32_t* __restrict__ cell_start, uint32_t* __restrict__ n_in_world) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (n_ptr) n = min(n, *n_ptr);
    if (i > n) return;
    // position i: keys (prev, cur]; prev = -1 at i == 0; cur = C+1 at i == n
    const int64_t prev = i == 0 ? -1 : (int64_t)sorted_key[i - 1];
    const int64_t cur = i == n ? (int64_t)cells + 1 : (int64_t)sorted_key[i];
    for (int64_t c = prev + 1; c <= cur; c++) {
        cell_start[c] = i;
        if (c == (int64_t)cells) *n_in_world = i;  // entities with a valid cell precede the key == cells tail
    }
}

// float -> double widening of a position upload (chd_set_entities_f32): channeld's entity positions arrive as unrealpb.FVector
// (three floats, pkg/unrealpb/unreal_common.proto:55-59) and become SpatialInfo doubles by float64(*vec.X)
// (pkg/unrealpb/extension.go:10-24).  That conversion is exact, so doing it here instead of on the host halves the bytes a
// position snapshot costs on PCIe without changing a single result bit.
__global__ void __launch_bounds__(256) widen_positions_kernel(const float* __restrict__ xf, const float* __restrict__ zf, double* x, double* z, uint32_t n) {
    const uint32_t i4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4u;
    if (i4 >= n) return;
    if (i4 + 4 <= n) {  // cudaMalloc'd buffers: 16-byte aligned at i4
        const float4 a = *reinterpret_cast<const float4*>(xf + i4), b = *reinterpret_cast<const float4*>(zf + i4);
        *reinterpret_cast<double2*>(x + i4) = make_double2((double)a.x, (double)a.y);
        *reinterpret_cast<double2*>(x + i4 + 2) = make_double2((double)a.z, (double)a.w);
        *reinterpret_cast<double2*>(z + i4) = make_double2((double)b.x, (double)b.y);
        *reinterpret_cast<double2*>(z + i4 + 2) = make_double2((double)b.z, (double)b.w);
    } else {
        for (uint32_t i = i4; i < n; i++) {
            x[i] = (double)xf[i];
            z[i] = (double)zf[i];
        }
    }
}

}  // namespace chd
