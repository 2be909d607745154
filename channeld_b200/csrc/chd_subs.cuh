// chd_subs.cuh — explicit subscriptions (SubscribeToChannel / UnsubscribeFromChannel, subscription.go:34-125) applied to the
// (subscriber, cell) pair state for a batch of ops: validate, sort the ops by (slot, cell), merge each touched slot's sorted op run
// into its sorted pair run, scan the new run lengths, write the new pair buffer.  Semantics: include/chd_gpu_subs.h.
#pragma once
#include "chd_types.cuh"
#include "../../include/chd_gpu_subs_sharded.h"

namespace chd {

// The uploaded batch (engine scratch).  Arrays of fields no op carries are nullptr; a present bit whose array is nullptr reads
// as absent.
struct SubOps {
    uint32_t n;
    const uint32_t *slot, *channel;
    const uint8_t *op, *present;
    const uint32_t* interval;
    const int32_t* delay;
    const uint8_t *skip_self, *skip_first;
};

// What the per-slot merge reads besides the pair runs: the ops in (slot, cell) order (idx[i] = op index), each op's slot (S when
// the op was rejected) and cell index, and where the statuses go.
struct SubMerge {
    SubOps ops;
    const uint32_t* __restrict__ idx;
    const uint32_t* __restrict__ eff_slot;
    const uint32_t* __restrict__ cell;
    uint8_t* __restrict__ status;
    uint32_t default_interval_ms;
    int32_t default_delay_ms;
    uint32_t id_start;
    int64_t now_ns;
    const int64_t* __restrict__ cell_start_ns;  // nullptr: one shared origin
    uint32_t* __restrict__ cell_max_interval;
};

constexpr uint32_t SUB_UNTOUCHED = 0xFFFFFFFFu;

// 1. statuses of the rejected ops; sort keys: the cell (C for a rejected op, sorted behind every valid one) and the slot (S).
// Slab (chd_apply_subscriptions_sharded): a SUB of a cell in a column the slab does not serve is rejected as well (after the slot
// and channel tests); an UNSUB of any cell is not.
template <bool Slab>
__global__ void __launch_bounds__(256) subs_validate_kernel(SubOps ops, uint32_t n_slots, const GridDev g, const uint32_t* __restrict__ conn_id,
                                                            const uint8_t* __restrict__ slot_ctl, uint32_t* __restrict__ key_cell,
                                                            uint32_t* __restrict__ eff_slot, uint32_t* __restrict__ cell, uint8_t* __restrict__ status) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ops.n) return;
    const uint32_t s = ops.slot[i], ch = ops.channel[i];
    const uint32_t cells = g.cells, id_start = g.id_start;
    // a free slot (never added, or released: connection id 0) or one with a removal / migration pending
    const bool slot_ok = s < n_slots && conn_id[s] != 0u && (!slot_ctl || slot_ctl[s] == SLOT_NORMAL);
    const bool ch_ok = ch >= id_start && ch - id_start < cells;
    const bool served = !Slab || (ops.op[i] & 1u) || !ch_ok || g.serves_column((ch - id_start) % g.cols);
    const bool ok = slot_ok && ch_ok && served;
    if (!ok) status[i] = !slot_ok ? (uint8_t)CHD_SUB_ERR_SLOT : (Slab && ch_ok) ? (uint8_t)CHD_SUB_ERR_OUTSIDE_SLAB : (uint8_t)CHD_SUB_ERR_CHANNEL;
    key_cell[i] = ok ? ch - id_start : cells;
    eff_slot[i] = ok ? s : n_slots;
    cell[i] = ok ? ch - id_start : 0u;
}

// 2. the second sort pass's keys: the slot of each op in the order of the first pass
__global__ void __launch_bounds__(256) subs_gather_kernel(const uint32_t* __restrict__ idx, uint32_t n, const uint32_t* __restrict__ eff_slot,
                                                          uint32_t* __restrict__ key) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) key[i] = eff_slot[idx[i]];
}

// One slot's merge of its previous pair run [pb, pe) (sorted by cell) with its op run from sorted position i0 (sorted by cell,
// array order within a cell).  Each group of ops on one cell starts from the pair the run holds there (if any) and applies the ops
// in order.  Count mode (WRITE == false) writes the statuses and returns the new run length; write mode writes the run at `o` and
// raises maxFanOutIntervalMs for every subscription it creates (subscription.go:84-86).
template <bool WRITE>
__device__ uint32_t subs_merge(const SubMerge& m, uint32_t s, uint32_t i0, const PairBuf& prev, uint32_t pb, uint32_t pe, const PairBuf& cur,
                               uint32_t o, uint32_t* __restrict__ pair_channel) {
    const SubOps& ops = m.ops;
    uint32_t i = i0, pp = pb, len = 0;
    auto op_cell = [&](uint32_t k) -> uint32_t {
        return (k < ops.n && m.eff_slot[m.idx[k]] == s) ? m.cell[m.idx[k]] : 0xFFFFFFFFu;
    };
    for (;;) {
        const uint32_t c_op = op_cell(i);
        const uint32_t c_pr = pp < pe ? prev.cell[pp] : 0xFFFFFFFFu;
        if (c_op == 0xFFFFFFFFu && c_pr == 0xFFFFFFFFu) break;
        bool ex = false;
        uint32_t dist = 0, interval = 0;
        uint8_t flags = 0;
        int64_t last = 0;
        uint64_t li = 0;
        uint32_t c;
        if (c_pr < c_op || c_pr == c_op) {  // the run's pair on this cell: the starting state
            c = c_pr;
            ex = true;
            dist = prev.dist[pp]; interval = prev.interval[pp]; flags = prev.flags[pp]; last = prev.last[pp]; li = prev.last_index[pp];
            pp++;
        } else {
            c = c_op;
        }
        for (; op_cell(i) == c; i++) {
            const uint32_t k = m.idx[i];
            const uint8_t pres = ops.present ? ops.present[k] : (uint8_t)0;
            const bool has_iv = (pres & CHD_SUBOPT_INTERVAL) && ops.interval, has_ss = (pres & CHD_SUBOPT_SKIP_SELF) && ops.skip_self;
            uint8_t st;
            if (ops.op[k] & 1u) {  // UnsubscribeFromChannel (subscription.go:104-125)
                st = ex ? (uint8_t)CHD_SUB_UNSUBSCRIBED : (uint8_t)CHD_SUB_NOT_SUBSCRIBED;
                ex = false;
            } else if (ex) {  // options merged, fan-out state untouched (subscription.go:44-57): delay / SkipFirst act at creation only
                if (has_iv) interval = ops.interval[k];
                if (has_ss) flags = ops.skip_self[k] ? (uint8_t)(flags | PF_SKIP_SELF) : (uint8_t)(flags & ~PF_SKIP_SELF);
                st = CHD_SUB_MERGED;
            } else {  // a new subscription (subscription.go:59-87): SPATIAL defaults, then the fields present
                interval = has_iv ? ops.interval[k] : m.default_interval_ms;
                const int32_t delay = ((pres & CHD_SUBOPT_DELAY) && ops.delay) ? ops.delay[k] : m.default_delay_ms;
                const bool ss = has_ss ? ops.skip_self[k] != 0 : true;
                const bool sf = ((pres & CHD_SUBOPT_SKIP_FIRST) && ops.skip_first) ? ops.skip_first[k] != 0 : false;
                flags = (uint8_t)((ss ? PF_SKIP_SELF : 0) | (sf ? PF_HAD_FIRST : 0));
                last = m.now_ns - (m.cell_start_ns ? m.cell_start_ns[c] : 0ll) + (int64_t)delay * 1000000ll;  // ch.GetTime().OffsetMs(delay)
                li = 0;
                dist = CHD_DIST_EXPLICIT;
                ex = true;
                st = CHD_SUB_NEW;
                if (WRITE && m.cell_max_interval[c] < interval) atomicMax(&m.cell_max_interval[c], interval);
            }
            if (!WRITE) m.status[k] = st;
        }
        if (!ex) continue;
        if (WRITE) {
            cur.sub[o] = s; cur.cell[o] = c; pair_channel[o] = c + m.id_start; cur.dist[o] = dist; cur.interval[o] = interval;
            cur.flags[o] = flags; cur.last[o] = last; cur.last_index[o] = li;
            o++;
        }
        len++;
    }
    return len;
}

// 3. the first op of each touched slot: marks the slot (beg = its first sorted position) and counts its new run
__global__ void __launch_bounds__(128) subs_count_kernel(SubMerge m, PairBuf prev, uint32_t n_slots, uint32_t* __restrict__ beg,
                                                         uint32_t* __restrict__ cnt) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m.ops.n) return;
    const uint32_t s = m.eff_slot[m.idx[i]];
    if (s >= n_slots || (i > 0 && m.eff_slot[m.idx[i - 1]] == s)) return;
    beg[s] = i;
    cnt[s] = subs_merge<false>(m, s, i, prev, prev.off[s], prev.off[s + 1], prev, 0, nullptr);
}

// 4. scan input: the new run length of slot s
struct SubCountIn {
    const uint32_t* beg;
    const uint32_t* cnt;
    const uint32_t* prev_off;
    __device__ __forceinline__ uint64_t operator()(uint64_t s) const { return beg[s] != SUB_UNTOUCHED ? cnt[s] : prev_off[s + 1] - prev_off[s]; }
};

// 5. the new pair buffer, one warp per slot: an untouched slot's run is copied by the whole warp (this pass streams every pair),
// a touched slot's merge is written by lane 0.  If the new total does not fit, NOTHING changes: every run is copied, every valid op
// gets CHD_SUB_ERR_CAPACITY and CHD_OVF_PAIRS is raised (the interest update's transactional rule).
constexpr int SUB_WRITE_THREADS = 256;
__global__ void __launch_bounds__(SUB_WRITE_THREADS) subs_write_kernel(SubMerge m, PairBuf prev, PairBuf cur, uint32_t n_slots, const uint32_t* __restrict__ noff,
                                                                       uint64_t pair_cap, const uint32_t* __restrict__ beg,
                                                                       uint32_t* __restrict__ pair_channel, Counters* __restrict__ ctr) {
    const uint64_t total = noff[n_slots];
    const bool ovf = total > pair_cap;
    const uint64_t gt = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gt == 0) {
        ctr->n_pairs = ovf ? (unsigned long long)prev.off[n_slots] : total;
        ctr->required_pairs = total;
        if (ovf) atomicOr(&ctr->overflow, (uint32_t)CHD_OVF_PAIRS);
        cur.off[n_slots] = ovf ? prev.off[n_slots] : (uint32_t)total;
    }
    const uint64_t s64 = gt >> 5;
    if (s64 >= n_slots) return;
    const uint32_t s = (uint32_t)s64, lane = threadIdx.x & 31;
    const uint32_t pb = prev.off[s], pe = prev.off[s + 1];
    const uint32_t o = ovf ? pb : noff[s];
    if (lane == 0) cur.off[s] = o;
    const uint32_t b = beg[s];
    if (b == SUB_UNTOUCHED || ovf) {
        for (uint32_t j = lane; j < pe - pb; j += 32) {
            const uint32_t p = pb + j, q = o + j;
            cur.sub[q] = s; cur.cell[q] = prev.cell[p]; pair_channel[q] = prev.cell[p] + m.id_start; cur.dist[q] = prev.dist[p];
            cur.interval[q] = prev.interval[p]; cur.flags[q] = prev.flags[p]; cur.last[q] = prev.last[p]; cur.last_index[q] = prev.last_index[p];
        }
        if (b != SUB_UNTOUCHED)  // (ovf) the slot's ops form one contiguous sorted run from b
            for (uint32_t i = b + lane; i < m.ops.n && m.eff_slot[m.idx[i]] == s; i += 32) m.status[m.idx[i]] = CHD_SUB_ERR_CAPACITY;
        return;
    }
    if (lane == 0) subs_merge<true>(m, s, b, prev, pb, pe, cur, o, pair_channel);
}

}  // namespace chd
