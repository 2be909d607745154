// chd_classes.cuh — window classes of a tick's due list (SURVEY.md §8f rank 1): the reference accumulates a fresh
// proto.Merge of the selected update window for EVERY subscriber (data.go:248-252) even when windows coincide.  The
// fan-out kernel tags every decision with its payload identity (DueKey, chd_fanout.cuh); here decisions with equal
// (channel, window, self-skip) identity are grouped so the host merges and frames each distinct payload once:
//   class_of[i]   dense class id of due record i
//   class_rep[k]  lowest due index of class k  (the record whose window the host merges)
//   class_cnt[k]  members of class k
// Grouping = open-addressing hash table keyed by the full 192-bit identity (window_hi, lo, word): a slot is claimed with
// one atomicCAS by the first record that reaches it and identified by THAT record's key from then on, so equal keys
// always meet in the same slot and unequal keys never share one — exact, no reliance on hash quality.
// A CHD_DUE_VOID hole (a slot an overflowed fan-out reserved but did not fill, chd_fanout.cuh) is not a decision: its key and
// window are whatever an earlier tick left there, so it probes nothing, gets class_of = CHD_DUE_VOID and is in no class.
#pragma once
#include "chd_types.cuh"

namespace chd {

__device__ __forceinline__ uint64_t class_mix(uint64_t x) {  // splitmix64 finaliser
    x ^= x >> 30; x *= 0xBF58476D1CE4E5B9ull;
    x ^= x >> 27; x *= 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

__global__ void __launch_bounds__(256)
    class_insert_kernel(const chd_due* __restrict__ due, const DueKey* __restrict__ key, const uint32_t* __restrict__ n_due_ptr, uint32_t due_cap,
                        uint32_t* __restrict__ table, uint32_t table_mask, uint32_t* __restrict__ slot_of, uint32_t* __restrict__ rep_min,
                        uint32_t* __restrict__ cnt) {
    const uint32_t n = min(*n_due_ptr, due_cap);
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (due[i].kind == CHD_DUE_VOID) {
        slot_of[i] = CHD_DUE_VOID;
        return;
    }
    const int64_t hi = due[i].window_hi;
    const DueKey k = key[i];
    const bool full = !((k.word >> 33) & 1ull);  // FULL sends of a channel share one payload whatever their window
    const int64_t khi = full ? 0ll : hi;
    uint32_t h = (uint32_t)class_mix(class_mix((uint64_t)khi) ^ class_mix((uint64_t)k.lo + 0x9E3779B97F4A7C15ull) ^ k.word) & table_mask;
    for (;;) {
        uint32_t owner = ((volatile uint32_t*)table)[h];
        if (owner == 0xFFFFFFFFu) {
            owner = atomicCAS(&table[h], 0xFFFFFFFFu, i);
            if (owner == 0xFFFFFFFFu) owner = i;  // claimed: this record's key names the slot
        }
        bool same = owner == i;
        if (!same) {
            const DueKey ko = key[owner];
            const bool ofull = !((ko.word >> 33) & 1ull);
            same = ko.word == k.word && ko.lo == k.lo && (ofull ? 0ll : due[owner].window_hi) == khi;
        }
        if (same) {
            slot_of[i] = h;
            atomicMin(&rep_min[h], i);
            atomicAdd(&cnt[h], 1u);
            return;
        }
        h = (h + 1) & table_mask;  // the table has >= 2 n slots: terminates
    }
}

__global__ void __launch_bounds__(256)
    class_flag_kernel(const uint32_t* __restrict__ n_due_ptr, uint32_t due_cap, const uint32_t* __restrict__ slot_of,
                      const uint32_t* __restrict__ rep_min, uint32_t* __restrict__ flag, unsigned long long* bump_epoch) {
    const uint32_t n = min(*n_due_ptr, due_cap);
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) *bump_epoch = chd_next_epoch(*bump_epoch);
    if (i < n) {
        const uint32_t h = slot_of[i];
        flag[i] = h != CHD_DUE_VOID && rep_min[h] == i ? 1u : 0u;
    }
}

// rank[] = exclusive scan of flag[]: class ids are numbered by their lowest member
__global__ void __launch_bounds__(256)
    class_finish_kernel(const uint32_t* __restrict__ n_due_ptr, uint32_t due_cap, const uint32_t* __restrict__ slot_of,
                        const uint32_t* __restrict__ rep_min, const uint32_t* __restrict__ cnt, const uint32_t* __restrict__ rank,
                        uint32_t* __restrict__ class_of, uint32_t* __restrict__ class_rep, uint32_t* __restrict__ class_cnt) {
    const uint32_t n = min(*n_due_ptr, due_cap);
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t h = slot_of[i];
    if (h == CHD_DUE_VOID) {
        class_of[i] = CHD_DUE_VOID;
        return;
    }
    const uint32_t rep = rep_min[h], id = rank[rep];
    class_of[i] = id;
    if (rep == i) {
        class_rep[id] = i;
        class_cnt[id] = cnt[h];
    }
}

}  // namespace chd
