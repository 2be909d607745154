// chd_shard.cuh — multi-GPU X-slab sharding kernels (SURVEY.md §8e): border export / halo import records.
#pragma once
#include "chd_types.cuh"

namespace chd {

// ---- X-slab sharding (SURVEY.md §8e).  A record is (global entity id, cell index).
// Border export and halo import are single-pass stream compactions (compact_1p, chd_scan.cuh): one launch each, input order kept.

// An own entity is exported when another rank may need it: its column is not strictly interior to this slab.
struct BorderFlag {
    GridDev g;
    const uint32_t* __restrict__ key;
    __device__ __forceinline__ bool operator()(uint64_t i) const {
        const uint32_t k = key[i];
        if (k >= g.cells) return false;
        const uint32_t col = k % g.cols;
        const bool interior = col >= g.col_lo + g.halo && col + g.halo < g.col_hi;
        if (interior) return false;
        // columns near a world edge with no neighbour beyond need no export
        const bool left_edge_open = g.col_lo > 0, right_edge_open = g.col_hi < g.cols;
        const bool near_left = col < g.col_lo + g.halo, near_right = col + g.halo >= g.col_hi;
        return (near_left && left_edge_open) || (near_right && right_edge_open) || col < g.col_lo || col >= g.col_hi;
    }
};
struct BorderSink {
    const uint32_t* __restrict__ key;
    EntityIds ids;
    uint32_t* __restrict__ out;
    uint32_t cap;
    uint32_t* __restrict__ count_out;
    Counters* __restrict__ ctr;
    __device__ __forceinline__ void operator()(uint64_t i, uint32_t k) const {
        if (k < cap) {
            out[2 * k] = ids.at((uint32_t)i);
            out[2 * k + 1] = key[i];
        }
    }
    __device__ __forceinline__ void total(uint32_t c) const {
        *count_out = c;
        if (c > cap) atomicOr(&ctr->overflow, (uint32_t)CHD_OVF_BORDER);
    }
};

// Gathered records: rank r's `per_rank` records start at word r * stride_words (the rest of a rank's contribution is its
// migration blob); with stride_words == 2 * per_rank the records are simply contiguous.
struct RecView {
    const uint32_t* base;
    uint32_t per_rank;
    uint64_t stride_words;
    __device__ __forceinline__ const uint32_t* at(uint64_t i) const {
        return base + (i / per_rank) * stride_words + 2ull * (i % per_rank);
    }
};

// keep gathered records whose column lies in this rank's extended range and which another rank exported.  `counts` (peer
// exchange) = live records per rank; without it the unused tail of a rank's records is padded with 0xFFFFFFFF (cell >= g.cells).
struct HaloFlag {
    GridDev g;
    RecView rec;
    const uint32_t* __restrict__ counts;
    uint32_t skip_first, skip_count;
    __device__ __forceinline__ bool operator()(uint64_t i) const {
        if (counts && (uint32_t)(i % rec.per_rank) >= counts[i / rec.per_rank]) return false;
        if (i >= skip_first && i - skip_first < skip_count) return false;
        const uint32_t cell = rec.at(i)[1];
        return cell < g.cells && g.serves_column(cell % g.cols);
    }
};
// appends the kept records after the `base` own entities and publishes the build length (own + halo) on the device:
// the host never needs the halo count, so the whole multi-GPU tick is free of host round trips.
struct HaloSink {
    RecView rec;
    uint32_t base, cap_total;
    uint32_t* __restrict__ key;
    uint32_t* __restrict__ gid;
    uint32_t* __restrict__ n_build;
    Counters* __restrict__ ctr;
    __device__ __forceinline__ void operator()(uint64_t i, uint32_t k) const {
        const uint64_t o = (uint64_t)base + k;
        if (o >= cap_total) return;
        const uint32_t* r = rec.at(i);
        gid[o] = r[0];
        key[o] = r[1];
    }
    __device__ __forceinline__ void total(uint32_t c) const {
        const uint64_t tot = (uint64_t)base + c;
        if (tot > cap_total) atomicOr(&ctr->overflow, (uint32_t)CHD_OVF_BORDER);
        *n_build = (uint32_t)min(tot, (uint64_t)cap_total);
    }
};

// ---- ring limits on slabs (include/chd_gpu_rings.h).  L = maxFanOutIntervalMs per cell (d_cell_max_interval), raised by this
// rank's interest updates; X = its exported shadow.  Records are (cell, value) pairs of u32.
// Export: (c, L[c]) for every served cell with L[c] > X[c], then X[c] = L[c] (ring_limit_advance_kernel, only if the records fit).
// Import: L[c] = max(L[c], v) and X[c] = max(X[c], v) for every gathered record (c, v).
// Claim: after an exchange in which every rank exports and then imports every record, each rank serving c holds M = max_r L_r[c] as
// of the exports.  Proof: X_r <= L_r always (both rise together on import, X is set to L on export).  Every value ever written to
// some X_s[c] was either exported by s or imported by s, and so was exported in some exchange; every rank serving c imported it
// there and L never falls, so every such rank holds L >= it.  Now take the rank s with L_s[c] = M at this export: if L_s[c] > X_s[c]
// it exports M now and every rank imports it; otherwise M = X_s[c] and the first sentence covers it.  Nothing above M is ever
// written, so every rank serving c ends at exactly M: the one-GPU value, since each (subscriber, cell) pair is created on the one
// rank that holds the subscriber, which serves every cell its query reaches.
struct RingLimitFlag {
    GridDev g;  // served columns: GridDev::serves_column
    const uint32_t* __restrict__ lim;
    const uint32_t* __restrict__ shadow;
    __device__ __forceinline__ bool operator()(uint64_t c) const { return g.serves_column((uint32_t)c % g.cols) && lim[c] > shadow[c]; }
};
struct RingLimitSink {
    const uint32_t* __restrict__ lim;
    uint32_t* __restrict__ out;
    uint32_t cap;
    uint32_t* __restrict__ count_out;
    Counters* __restrict__ ctr;  // nullptr: the caller reads the count and reports an overflow itself
    __device__ __forceinline__ void operator()(uint64_t c, uint32_t k) const {
        if (k < cap) {
            out[2 * k] = (uint32_t)c;
            out[2 * k + 1] = lim[c];
        }
    }
    __device__ __forceinline__ void total(uint32_t n) const {
        *count_out = n;
        if (n > cap && ctr) atomicOr(&ctr->overflow, (uint32_t)CHD_OVF_BORDER);
    }
};
// X[c] = exported value, for every exported record; nothing if the export did not fit (it is repeated in full next time)
__global__ void __launch_bounds__(256) ring_limit_advance_kernel(const uint32_t* __restrict__ rec, const uint32_t* __restrict__ count, uint32_t cap,
                                                                 uint32_t* __restrict__ shadow) {
    const uint32_t n = *count, k = blockIdx.x * blockDim.x + threadIdx.x;
    if (n > cap || k >= n) return;
    shadow[rec[2 * k]] = rec[2 * k + 1];
}

// Gathered ring-limit records: rank r's section starts at word r * stride_words of `base`.  headed: the section is [count, 3 words of
// padding, records] (chd_tick_sharded's contribution); otherwise `base` holds per_rank records of one rank, all live.
struct RingLimitView {
    const uint32_t* base;
    uint32_t per_rank;
    uint64_t stride_words;
    bool headed;
};
__global__ void __launch_bounds__(256) ring_limit_import_kernel(RingLimitView v, uint32_t ranks, uint32_t cells, uint32_t* __restrict__ lim,
                                                                uint32_t* __restrict__ shadow) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (uint64_t)ranks * v.per_rank) return;
    const uint32_t r = (uint32_t)(i / v.per_rank), k = (uint32_t)(i % v.per_rank);
    const uint32_t* sec = v.base + r * v.stride_words;
    if (v.headed && k >= min(sec[0], v.per_rank)) return;
    const uint32_t* rec = sec + (v.headed ? 4 : 0) + 2ull * k;
    const uint32_t c = rec[0], val = rec[1];
    if (c >= cells) return;
    if (lim[c] < val) atomicMax(&lim[c], val);
    if (shadow[c] < val) atomicMax(&shadow[c], val);
}

// ---- the exchange itself over peer memory (NVLink): no collective library call on the tick path.
// Every rank owns a WINDOW = 2 buffers (tick parity) x world x stride words + 2 x world 64-bit flags, mapped into every peer with
// CUDA IPC at chd_comm_init.  peer_push_kernel copies this rank's live border records (and its migration blob) straight into
// slot [parity][rank] of every peer's window, then publishes (sequence << 32 | record count) in the peer's flag [parity][rank]
// (system-scope release: data first, fence, the last block writes the flags).  peer_wait_kernel on the receiving side polls its
// OWN flags until all `world` contributions of this sequence have landed (acquire) and hands the counts to the import.
// Double buffering is enough without any further handshake: a peer can only push tick k+2 into buffer k%2 after it has imported
// tick k+1, which needed this rank's push of k+1, which this rank issued after its own import of tick k (stream order).
constexpr int CHD_MAX_PEERS = 16;
struct PeerWindows {
    uint32_t* base[CHD_MAX_PEERS];
};
__device__ __forceinline__ unsigned long long* peer_flags(uint32_t* win_base, uint64_t stride_words, uint32_t world) {
    return reinterpret_cast<unsigned long long*>(win_base + 2ull * world * stride_words);
}

// After the migration blob comes the ring-limit section ([count, 3 words of padding, records]): its header and live records move.
__global__ void __launch_bounds__(256) peer_push_kernel(const uint32_t* __restrict__ local, const uint32_t* __restrict__ count_ptr, uint32_t cap,
                                                        uint64_t blob_words, uint32_t ring_cap, uint64_t stride_words, PeerWindows peers, uint32_t world,
                                                        uint32_t rank, unsigned long long* __restrict__ seq_ctr, uint32_t* __restrict__ done_ctr,
                                                        unsigned long long* bump_epoch) {
    __shared__ bool s_last;
    const unsigned long long seq = *seq_ctr + 1ull;  // (the last block advances the counter after every block has read it)
    const uint32_t parity = (uint32_t)(seq & 1ull);
    const uint32_t count = min(*count_ptr, cap);
    const uint64_t rec_words = 2ull * count;
    const uint64_t rec_q = rec_words / 4, blob_q = blob_words / 4;  // 16-byte moves; the blob starts 16-byte aligned (cap is even)
    const uint64_t ring_off = 2ull * cap + blob_words;                // (16-byte aligned: blob_words is a multiple of 4)
    const uint64_t ring_q = (4ull + 2ull * min(local[ring_off], ring_cap) + 3ull) / 4;
    const uint64_t slot_off = ((uint64_t)parity * world + rank) * stride_words;
    const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, nthr = (uint64_t)gridDim.x * blockDim.x;
    for (uint32_t r = 0; r < world; r++) {
        uint32_t* dst = peers.base[r] + slot_off;
        const uint4* s4 = reinterpret_cast<const uint4*>(local);
        uint4* d4 = reinterpret_cast<uint4*>(dst);
        for (uint64_t i = tid; i < rec_q; i += nthr) d4[i] = s4[i];
        for (uint64_t i = rec_q * 4 + tid; i < rec_words; i += nthr) dst[i] = local[i];
        const uint4* b4 = reinterpret_cast<const uint4*>(local + 2ull * cap);
        uint4* e4 = reinterpret_cast<uint4*>(dst + 2ull * cap);
        for (uint64_t i = tid; i < blob_q; i += nthr) e4[i] = b4[i];
        const uint4* r4 = reinterpret_cast<const uint4*>(local + ring_off);
        uint4* q4 = reinterpret_cast<uint4*>(dst + ring_off);
        for (uint64_t i = tid; i < ring_q; i += nthr) q4[i] = r4[i];
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) s_last = atomicAdd(done_ctr, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!s_last) return;
    __threadfence_system();
    if (threadIdx.x < world) {
        volatile unsigned long long* f = peer_flags(peers.base[threadIdx.x], stride_words, world) + (uint64_t)parity * world + rank;
        *f = (seq << 32) | (unsigned long long)count;
    }
    if (threadIdx.x == 0) {
        *done_ctr = 0;
        *seq_ctr = seq;
        if (bump_epoch) *bump_epoch = chd_next_epoch(*bump_epoch);  // the import's compaction site
    }
}

// one block, one thread per rank; bounded wait (a peer that never arrives must surface as an error, never as a hung GPU)
__global__ void peer_wait_kernel(uint32_t* own_win, uint64_t stride_words, uint32_t world, const unsigned long long* __restrict__ seq_ctr,
                                 uint32_t* __restrict__ counts, Counters* __restrict__ ctr) {
    const uint32_t r = threadIdx.x;
    if (r >= world) return;
    const unsigned long long seq = *seq_ctr;  // this rank's push of the same tick has completed (stream order)
    volatile unsigned long long* f = peer_flags(own_win, stride_words, world) + (seq & 1ull) * world + r;
    unsigned long long t0 = 0, v = 0;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    for (;;) {
        v = *f;
        if ((v >> 32) == (seq & 0xFFFFFFFFull)) break;
        unsigned long long t1;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        if (t1 - t0 > 20000000000ull) {  // 20 s: ranks may reach a tick far apart (host-side work between ticks); still never a hung GPU
            atomicOr(&ctr->overflow, (uint32_t)CHD_OVF_BORDER | 0x80000000u);
            v = 0;
            break;
        }
        __nanosleep(200);
    }
    __threadfence_system();
    counts[r] = (uint32_t)v;
}

// chd_get_rehome: own entities whose column now belongs to another rank (a set: block-aggregated append)
__global__ void __launch_bounds__(256) rehome_kernel(GridDev g, const uint32_t* __restrict__ key, EntityIds ids, uint32_t n,
                                                     uint32_t world, uint32_t* __restrict__ out_gid, uint32_t* __restrict__ out_rank,
                                                     uint32_t cap, uint32_t* __restrict__ count) {
    __shared__ uint32_t s_cnt, s_base;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    bool away = false;
    uint32_t col = 0, my = 0;
    if (i < n && key[i] < g.cells) {
        col = key[i] % g.cols;
        away = col < g.col_lo || col >= g.col_hi;
    }
    if (away) my = atomicAdd(&s_cnt, 1u);
    __syncthreads();
    if (threadIdx.x == 0 && s_cnt) s_base = atomicAdd(count, s_cnt);
    __syncthreads();
    if (away && s_base + my < cap) {
        out_gid[s_base + my] = ids.at(i);
        out_rank[s_base + my] = slab_owner(col, g.cols, world);
    }
}

__global__ void __launch_bounds__(256) slot_ctl_mark_kernel(const uint32_t* __restrict__ slot, uint32_t n, uint8_t ctl, uint8_t* __restrict__ slot_ctl) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) slot_ctl[slot[i]] = ctl;
}
// chd_migrate_in: slot[i] becomes connection conn[i]; its previous run is record (first_index + i) of src_rank's blob
__global__ void __launch_bounds__(256) slot_import_mark_kernel(const uint32_t* __restrict__ slot, const uint32_t* __restrict__ conn, uint32_t n,
                                                               uint32_t src_rank, uint32_t first_index, uint8_t* __restrict__ slot_ctl,
                                                               uint32_t* __restrict__ slot_src, uint32_t* __restrict__ conn_id) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t s = slot[i];
    slot_ctl[s] = SLOT_IMPORT;
    slot_src[s] = (src_rank << 20) | ((first_index + i) & 0xFFFFFu);
    conn_id[s] = conn[i];
}

// chd_migrate_out: packs the subscriptions + fan-out state of the listed slots into this rank's migration blob (MigView layout).
// One block: the lists are control-plane sized (a per-cent of the subscribers cross a slab boundary per tick).
__global__ void __launch_bounds__(256) mig_pack_kernel(const uint32_t* __restrict__ slot, uint32_t n, PairBuf pb, const uint32_t* __restrict__ conn_id,
                                                       uint32_t* __restrict__ blob, MigView lay, Counters* __restrict__ ctr) {
    __shared__ uint32_t s_warp[8], s_run;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_run = 0;
    __syncthreads();
    uint32_t* off = blob + lay.o_off();
    uint32_t* oconn = blob + lay.o_conn();
    uint32_t *ocell = blob + lay.o_cell(), *odist = blob + lay.o_dist(), *oiv = blob + lay.o_interval(), *ofl = blob + lay.o_flags();
    int64_t* olast = reinterpret_cast<int64_t*>(blob + lay.o_last());
    uint64_t* olidx = reinterpret_cast<uint64_t*>(blob + lay.o_lidx());
    const uint32_t n_fit = min(n, lay.max_subs);
    for (uint32_t base = 0; base < n_fit; base += blockDim.x) {
        const uint32_t i = base + threadIdx.x;
        uint32_t s = 0, p0 = 0, k = 0;
        if (i < n_fit) {
            s = slot[i];
            p0 = pb.off[s];
            k = pb.off[s + 1] - p0;
        }
        uint32_t incl = k;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t a = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += a;
        }
        if (lane == 31) s_warp[w] = incl;
        __syncthreads();
        uint32_t o = s_run + incl - k;
        for (int j = 0; j < w; j++) o += s_warp[j];
        if (i < n_fit) {
            off[i] = o;
            oconn[i] = conn_id[s];
            for (uint32_t j = 0; j < k && o + j < lay.max_pairs; j++) {
                ocell[o + j] = pb.cell[p0 + j]; odist[o + j] = pb.dist[p0 + j]; oiv[o + j] = pb.interval[p0 + j];
                ofl[o + j] = pb.flags[p0 + j]; olast[o + j] = pb.last[p0 + j]; olidx[o + j] = pb.last_index[p0 + j];
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t tot = 0;
            for (int j = 0; j < 8; j++) tot += s_warp[j];
            s_run += tot;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        off[n_fit] = s_run;
        blob[0] = n_fit;
        blob[1] = min(s_run, lay.max_pairs);
        if (n > lay.max_subs || s_run > lay.max_pairs) atomicOr(&ctr->overflow, (uint32_t)CHD_OVF_BORDER);  // truncated: those arrive without state
    }
}

}  // namespace chd
