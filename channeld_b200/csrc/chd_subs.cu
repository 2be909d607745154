// chd_subs.cu — explicit subscriptions to spatial channels (include/chd_gpu_subs.h, and on slabs include/chd_gpu_subs_sharded.h):
// a stage of its own on the engine stream, between ticks.  Kernels: chd_subs.cuh.
#include "chd_engine.h"

#include "chd_subs.cuh"

namespace {

// the op arrays hold `need` ops (grown together; contents are not kept)
bool subs_reserve(chd_engine* e, uint64_t need) {
    chd_engine::Subs& x = e->subs;
    if (!x.beg) {
        const uint64_t S = e->lim.max_subscribers;
        if (!(dalloc(e, &x.beg, S) && dalloc(e, &x.cnt, S) && dalloc(e, &x.noff, S + 2))) return false;
    }
    if (need <= x.op_cap) return true;
    const uint64_t count = std::min<uint64_t>(e->lim.max_pairs, std::max<uint64_t>(need + need / 2, 1024));
    bool ok = true;
    auto grow = [&](auto** p) {
        uint64_t cap = x.op_cap;
        ok = ok && ensure_cap(e, p, &cap, need, count);
    };
    grow(&x.slot); grow(&x.channel); grow(&x.interval); grow(&x.delay); grow(&x.op); grow(&x.present); grow(&x.skip_self);
    grow(&x.skip_first); grow(&x.status); grow(&x.key); grow(&x.key_out); grow(&x.idx1); grow(&x.idx2); grow(&x.eff_slot); grow(&x.cell);
    if (ok) x.op_cap = count;
    return ok;
}

template <typename T>
chd_status upload(chd_engine* e, T* dst, const T* src, uint32_t n, const T** view) {
    *view = nullptr;
    if (!src) return CHD_OK;
    CU(e, cudaMemcpyAsync(dst, src, sizeof(T) * n, cudaMemcpyDefault, e->stream));
    *view = dst;
    return CHD_OK;
}

// a new epoch of the query stage's scan sites (the pair sort's and the slot scan's), one per use of a site
void open_epoch(chd_engine* e, cudaStream_t s) {
    chd_epoch_tick(e, s, EP_QUERY);
    bump_epoch_kernel<<<1, 1, 0, s>>>(e->d_epoch + EP_QUERY);
}

// the batch limits, checked after the call's rule: CHD_ERR_CAPACITY, nothing applied
chd_status check_batch(chd_engine* e, uint32_t n, const char* fn) {
    if (n > e->lim.max_pairs) {
        e->fail("%s: %u ops > max_pairs %llu", fn, n, (unsigned long long)e->lim.max_pairs);
        return CHD_ERR_CAPACITY;
    }
    if (e->n_slots >= (1u << 20)) {  // the sort by slot takes <= 2 passes of <= 10-bit digits
        e->fail("%s: %u subscriber slots (at most 2^20 - 1)", fn, e->n_slots);
        return CHD_ERR_CAPACITY;
    }
    return CHD_OK;
}

// Both entry points after their rule, their checks and CHD_ENTER: `slab` rejects SUBs of cells the slab does not serve.
chd_status apply(chd_engine* e, const chd_sub_batch* b, int64_t now_ns, uint8_t* out_status, bool slab) {
    const uint32_t n = b->n;
    if (!subs_reserve(e, n)) return CHD_ERR_CUDA;
    chd_engine::Subs& x = e->subs;
    cudaStream_t s = e->stream;
    SubOps ops{};
    ops.n = n;
    chd_status st = CHD_OK;
    if ((st = upload(e, x.slot, b->slot, n, &ops.slot)) != CHD_OK || (st = upload(e, x.channel, b->channel_id, n, &ops.channel)) != CHD_OK ||
        (st = upload(e, x.op, b->op, n, &ops.op)) != CHD_OK || (st = upload(e, x.present, b->present, n, &ops.present)) != CHD_OK ||
        (st = upload(e, x.interval, b->interval_ms, n, &ops.interval)) != CHD_OK || (st = upload(e, x.delay, b->delay_ms, n, &ops.delay)) != CHD_OK ||
        (st = upload(e, x.skip_self, b->skip_self, n, &ops.skip_self)) != CHD_OK ||
        (st = upload(e, x.skip_first, b->skip_first, n, &ops.skip_first)) != CHD_OK)
        return st;
    const uint32_t S = e->n_slots, C = e->g.cells;
    // 1. validate
    const uint8_t* ctl = e->lifecycle_used ? e->d_slot_ctl : nullptr;
    if (slab)
        subs_validate_kernel<true><<<blocks_for(n, 256), 256, 0, s>>>(ops, S, e->g, e->d_conn, ctl, x.key, x.eff_slot, x.cell, x.status);
    else
        subs_validate_kernel<false><<<blocks_for(n, 256), 256, 0, s>>>(ops, S, e->g, e->d_conn, ctl, x.key, x.eff_slot, x.cell, x.status);
    KCHECK(e);
    if (S > 0) {
        PairBuf& prev = e->pairs[e->cur];
        PairBuf& cur = e->pairs[e->cur ^ 1];
        // 2. stable sort of the op indices by (slot, cell): by cell, then stably by slot (rejected ops last)
        chd_epoch_tick(e, s, EP_QUERY);
        st = chd_cell_sort(e, s, e->pair_sort, C + 1, x.key, nullptr, n, nullptr, x.key_out, x.idx1, nullptr, e->d_epoch + EP_QUERY);
        if (st != CHD_OK) return st;
        subs_gather_kernel<<<blocks_for(n, 256), 256, 0, s>>>(x.idx1, n, x.eff_slot, x.key);
        KCHECK(e);
        chd_epoch_tick(e, s, EP_QUERY);
        st = chd_cell_sort(e, s, e->pair_sort, S + 1, x.key, x.idx1, n, nullptr, x.key_out, x.idx2, nullptr, e->d_epoch + EP_QUERY);
        if (st != CHD_OK) return st;
        // 3. each touched slot's new run length (and the statuses)
        const SubMerge m{ops, x.idx2, x.eff_slot, x.cell, x.status, e->g.default_interval_ms, e->g.default_delay_ms, e->g.id_start, now_ns,
                         e->have_cell_start ? e->d_cell_start_ns : nullptr, e->d_cell_max_interval};
        CU(e, cudaMemsetAsync(x.beg, 0xFF, sizeof(uint32_t) * S, s));
        subs_count_kernel<<<blocks_for(n, 128), 128, 0, s>>>(m, prev, S, x.beg, x.cnt);
        KCHECK(e);
        // 4. new offsets of every slot; the capacity decision is made on the device, by the write pass
        open_epoch(e, s);
        KCHECK(e);
        SCAN(e, exclusive_scan_fn<SubCountIn, uint32_t>(SubCountIn{x.beg, x.cnt, prev.off}, x.noff, S, e->site_slot, s));
        // 5. the new pair buffer
        subs_write_kernel<<<blocks_for((uint64_t)S * 32, SUB_WRITE_THREADS), SUB_WRITE_THREADS, 0, s>>>(m, prev, cur, S, x.noff, e->lim.max_pairs, x.beg,
                                                                                                      e->d_pair_ch, e->d_ctr);
        KCHECK(e);
        // 6. pairs grouped by cell for the fan-out pass, as the interest update groups them
        chd_epoch_tick(e, s, EP_QUERY);
        st = chd_cell_sort(e, s, e->pair_sort, C, cur.cell, nullptr, (uint32_t)e->lim.max_pairs, cur.off + S, nullptr, e->d_by_cell, nullptr,
                           e->d_epoch + EP_QUERY);
        if (st != CHD_OK) return st;
        // 7. the new buffer is the current one (after an overflow it holds the previous pairs unchanged)
        e->cur ^= 1;
        e->pair_ch_valid = true;
        e->by_cell_valid = true;
    }
    if (out_status) {
        CU(e, cudaMemcpyAsync(out_status, x.status, n, cudaMemcpyDefault, s));
        CU(e, cudaStreamSynchronize(s));
    }
    return CHD_OK;
}

}  // namespace

extern "C" {

chd_status chd_apply_subscriptions(chd_engine* e, const chd_sub_batch* b, int64_t now_ns, uint8_t* out_status) {
    if (!e || !b) return CHD_ERR_INVALID;
    const uint32_t n = b->n;
    if (n && (!b->slot || !b->channel_id || !b->op)) return CHD_ERR_INVALID;
    if (chd_rule_explicit_subs(e, "chd_apply_subscriptions") != CHD_OK) return CHD_ERR_STATE;
    const chd_status st = check_batch(e, n, "chd_apply_subscriptions");
    if (st != CHD_OK || n == 0) return st;
    // LOCK: this stage opens epochs of the query stage's scan sites, which chd_query_channel_ids (any thread) also bumps.
    // COPY_WAIT: the pair buffer written here is the one the pending copy kernel's tick will overwrite next.
    // FETCH_GUARD: the pairs, their channel ids and the by-cell grouping are read-back sources.
    CHD_ENTER(e, ENTRY_LOCK | ENTRY_COPY_WAIT | ENTRY_FETCH_GUARD);
    return apply(e, b, now_ns, out_status, false);
}

chd_status chd_apply_subscriptions_sharded(chd_engine* e, const chd_sub_batch* b, int64_t now_ns, uint8_t* out_status) {
    if (!e || !b) return CHD_ERR_INVALID;
    const uint32_t n = b->n;
    if (n && (!b->slot || !b->channel_id || !b->op)) return CHD_ERR_INVALID;
    const char* fn = "chd_apply_subscriptions_sharded";
    if (chd_rule_explicit_subs_slab(e, fn) != CHD_OK || chd_rule_rings_staged(e, fn) != CHD_OK) return CHD_ERR_STATE;
    const chd_status st = check_batch(e, n, fn);
    if (st != CHD_OK || n == 0) return st;
    // the needs of chd_apply_subscriptions, for the same reasons
    CHD_ENTER(e, ENTRY_LOCK | ENTRY_COPY_WAIT | ENTRY_FETCH_GUARD);
    return apply(e, b, now_ns, out_status, true);
}

}  // extern "C"
