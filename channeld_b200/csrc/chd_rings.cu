// chd_rings.cu — update rings: one tick's host-owned rings (set or prefetched), device-owned rings (ChannelData.OnUpdate's buffer
// maintenance on the GPU, data.go:149-173) with or without each update's bytes, and their read-back.
#include "chd_engine.h"

#include "chd_gpu_ring_bytes.h"
#include "chd_misc.cuh"
#include "chd_rings.cuh"

using Rings = chd_engine::Rings;

extern "C" {

// argument checks of one tick's host-owned rings (chd_set_rings / chd_prefetch_rings)
static chd_status check_rings(chd_engine* e, const char* fn, const uint32_t* ring_off, uint32_t n_entries, const int64_t* arrival, const uint32_t* sender,
                              const uint64_t* index) {
    if (!e || !ring_off) return CHD_ERR_INVALID;
    if (e->rings.owned) {
        e->fail("%s: the rings are device-owned (chd_rings_init): use chd_rings_append", fn);
        return CHD_ERR_STATE;
    }
    if (n_entries > e->lim.max_ring_entries) {
        e->fail("%u ring entries > max_ring_entries %u", n_entries, e->lim.max_ring_entries);
        return CHD_ERR_CAPACITY;
    }
    if (n_entries && (!arrival || !sender || !index)) return CHD_ERR_INVALID;
    return CHD_OK;
}

// copies one tick's host-owned rings into staging set `r` on `s`, with their entry count and whether they carry channel_msg_index
static chd_status copy_rings(chd_engine* e, cudaStream_t s, Rings::RStage& r, const uint32_t* ring_off, uint32_t n_entries, const int64_t* arrival,
                             const uint32_t* sender, const uint64_t* index, const uint64_t* ch_msg_index) {
    const uint64_t C = e->g.cells;
    CU(e, cudaMemcpyAsync(r.off, ring_off, sizeof(uint32_t) * (C + 1), cudaMemcpyDefault, s));
    if (n_entries) {
        CU(e, cudaMemcpyAsync(r.arrival, arrival, sizeof(int64_t) * n_entries, cudaMemcpyDefault, s));
        CU(e, cudaMemcpyAsync(r.sender, sender, sizeof(uint32_t) * n_entries, cudaMemcpyDefault, s));
        CU(e, cudaMemcpyAsync(r.index, index, sizeof(uint64_t) * n_entries, cudaMemcpyDefault, s));
    }
    if (ch_msg_index) CU(e, cudaMemcpyAsync(r.cmi, ch_msg_index, sizeof(uint64_t) * C, cudaMemcpyDefault, s));
    r.total = n_entries;
    r.has_cmi = ch_msg_index != nullptr;
    return CHD_OK;
}

// staged host-owned rings as the kernels read them: a CSR by cell
static RingDev staged_ring(const chd_engine* e, const Rings::RStage& r) {
    return RingDev{r.off, r.off + 1, r.arrival, r.sender, r.index, r.has_cmi ? r.cmi : nullptr, e->rings.d_total, nullptr};
}

static void pf_reader_reset(Rings& R) { R.pf.cur = -1, R.pf.wait = false; }  // the rings read are no prefetch set

chd_status chd_rings_create(chd_engine* e) {
    Rings& R = e->rings;
    const uint64_t C = e->g.cells, RE = e->lim.max_ring_entries;
    if (!(dalloc(e, &R.begin, C + 1) && dalloc(e, &R.end, C + 1) && dalloc(e, &R.flat_off, C + 2) && dalloc(e, &R.upd_off, C + 1) && dalloc(e, &R.d_total, 1) &&
          dalloc(e, &R.set.off, C + 1) && dalloc(e, &R.set.arrival, RE) && dalloc(e, &R.set.sender, RE) && dalloc(e, &R.set.index, RE) && dalloc(e, &R.set.cmi, C)))
        return CHD_ERR_CUDA;
    R.view = staged_ring(e, R.set);  // empty host-owned rings
    CU(e, cudaMemsetAsync(R.set.off, 0, (C + 1) * 4, e->stream));
    CU(e, cudaMemsetAsync(R.set.cmi, 0, C * 8, e->stream));
    CU(e, cudaMemsetAsync(R.d_total, 0, 4, e->stream));
    return CHD_OK;
}

chd_status chd_set_rings(chd_engine* e, const uint32_t* ring_off, uint32_t n_entries, const int64_t* arrival, const uint32_t* sender,
                         const uint64_t* index, const uint64_t* ch_msg_index) {
    chd_status st = check_rings(e, "chd_set_rings", ring_off, n_entries, arrival, sender, index);
    if (st != CHD_OK) return st;
    if (chd_rule_no_chain(e, "chd_set_rings", true) != CHD_OK) return CHD_ERR_STATE;
    CHD_ENTER(e, ENTRY_DEVICE);
    Rings& R = e->rings;
    const bool in_place = chd_is_device_ptr(e, ring_off) && (!n_entries || (chd_is_device_ptr(e, arrival) && chd_is_device_ptr(e, sender) && chd_is_device_ptr(e, index))) &&
                          (!ch_msg_index || chd_is_device_ptr(e, ch_msg_index));
    st = in_place ? CHD_OK : copy_rings(e, e->stream, R.set, ring_off, n_entries, arrival, sender, index, ch_msg_index);
    if (st != CHD_OK) return st;
    R.view = in_place ? RingDev{ring_off, ring_off + 1, arrival, sender, index, ch_msg_index, R.d_total, nullptr}  // consumed in place
                      : staged_ring(e, R.set);
    pf_reader_reset(R);
    // the fan-out kernel clamps ring_off to this: a lying caller cannot cause out-of-bounds reads
    R.total = n_entries;
    R.total_pending = true;
    return CHD_OK;
}

chd_status chd_prefetch_rings(chd_engine* e, const uint32_t* ring_off, uint32_t n_entries, const int64_t* arrival, const uint32_t* sender,
                              const uint64_t* index, const uint64_t* ch_msg_index) {
    chd_status st = check_rings(e, "chd_prefetch_rings", ring_off, n_entries, arrival, sender, index);
    if (st != CHD_OK) return st;
    CHD_ENTER(e, ENTRY_DEVICE);
    int set = 0;
    st = chd_pf_begin(e, e->rings.pf, &set);
    if (st != CHD_OK) return st;
    Rings::RStage& r = e->rings.pf_set[set];
    const uint64_t C = e->g.cells, R = e->lim.max_ring_entries;
    if (!r.cmi && !(dalloc(e, &r.off, C + 1) && dalloc(e, &r.arrival, R) && dalloc(e, &r.sender, R) && dalloc(e, &r.index, R) && dalloc(e, &r.cmi, C)))
        return CHD_ERR_CUDA;  // (cmi is allocated last)
    st = copy_rings(e, e->up_stream, r, ring_off, n_entries, arrival, sender, index, ch_msg_index);
    return st != CHD_OK ? st : chd_pf_end(e, e->rings.pf);
}

void chd_rings_adopt(chd_engine* e) {
    Rings& R = e->rings;
    if (!chd_pf_adopt(R.pf)) return;
    R.view = staged_ring(e, R.pf_set[R.pf.cur]);
    R.total = R.pf_set[R.pf.cur].total;
    R.total_pending = true;
}

chd_status chd_ring_total_flush(chd_engine* e, cudaStream_t s) {
    Rings& R = e->rings;
    if (!R.total_pending) return CHD_OK;
    set_u32_kernel<<<1, 1, 0, s>>>(R.d_total, R.total);
    KCHECK(e);
    R.total_pending = false;
    return CHD_OK;
}

RingDev chd_ring_view(const chd_engine* e) {
    RingDev ring = e->rings.view;
    ring.start = e->have_cell_start ? e->d_cell_start_ns : nullptr;
    return ring;
}

/* ---- device-owned rings: ChannelData.OnUpdate's buffer maintenance on the GPU (data.go:149-173) */

// One append on the engine stream: its updates into upd_* (with byte_off, their bytes into bytes.upd_*), then staged for
// chd_tick_sharded (a communicator engine) or applied
static chd_status rings_append_on(chd_engine* e, const uint32_t* upd_off, uint32_t n_updates, const int64_t* arrival_ns, const uint32_t* sender_conn_id,
                                  const uint64_t* byte_off = nullptr, const uint8_t* bytes = nullptr) {
    Rings& R = e->rings;
    Rings::RingBytes& rb = R.bytes;
    cudaStream_t s = e->stream;
    const uint32_t C = e->g.cells;
    const uint64_t grown = (uint64_t)n_updates + n_updates / 2 + 1024, nb = byte_off ? byte_off[n_updates] : 0;
    if ((byte_off && (!ensure_cap(e, &rb.upd_boff, &rb.upd_boff_cap, (uint64_t)n_updates + 1, grown + 1) ||
                      !ensure_cap(e, &rb.upd_bytes, &rb.upd_bytes_cap, nb + 1, nb + nb / 2 + 4096))) ||
        !ensure_cap(e, &R.upd_arrival, &R.upd_arrival_cap, n_updates, grown) || !ensure_cap(e, &R.upd_sender, &R.upd_sender_cap, n_updates, grown))
        return CHD_ERR_CUDA;
    CU(e, cudaMemcpyAsync(R.upd_off, upd_off, sizeof(uint32_t) * ((uint64_t)C + 1), cudaMemcpyDefault, s));
    if (n_updates) {
        CU(e, cudaMemcpyAsync(R.upd_arrival, arrival_ns, sizeof(int64_t) * n_updates, cudaMemcpyDefault, s));
        CU(e, cudaMemcpyAsync(R.upd_sender, sender_conn_id, sizeof(uint32_t) * n_updates, cudaMemcpyDefault, s));
    }
    if (byte_off) CU(e, cudaMemcpyAsync(rb.upd_boff, byte_off, 8 * ((uint64_t)n_updates + 1), cudaMemcpyHostToDevice, s));
    if (nb) CU(e, cudaMemcpyAsync(rb.upd_bytes, bytes, nb, cudaMemcpyDefault, s));
    R.appended = true;
    if (e->comm) {  // rule 12: chd_tick_sharded appends them once the other ranks' ring limits are in
        R.staged = true;
        R.staged_updates = n_updates;
        return CHD_OK;
    }
    return chd_rings_apply(e, s, n_updates);
}

// The live-entry CSR of the device-owned rings into flat_off on the engine stream (control-plane read-back: a plain two-pass scan
// through scratch that is free between ticks; the live lengths go through upd_off, which holds no staged append here: rule 12)
static chd_status live_entry_csr(chd_engine* e) {
    Rings& R = e->rings;
    cudaStream_t s = e->stream;
    const uint32_t C = e->g.cells;
    if (!R.scan_scratch && !dalloc(e, &R.scan_scratch, scan_scratch_elems(C + 1))) return CHD_ERR_CUDA;
    ring_len_kernel<<<blocks_for(C, 128), 128, 0, s>>>(C, R.begin, R.end, R.upd_off);
    KCHECK(e);
    SCAN(e, exclusive_scan<uint32_t, uint32_t>(R.upd_off, R.flat_off, C, R.scan_scratch, s));
    return CHD_OK;
}

chd_status chd_rings_init(chd_engine* e, uint32_t capacity_per_cell) {
    if (!e || capacity_per_cell <= RING_MAX_BUFFER) {
        if (e) e->fail("chd_rings_init: capacity_per_cell must exceed %u (MaxUpdateMsgBufferSize: the reference's buffer may grow beyond it)", RING_MAX_BUFFER);
        return CHD_ERR_INVALID;
    }
    if (chd_rule_no_chain(e, "chd_rings_init", false) != CHD_OK) return CHD_ERR_STATE;
    const uint64_t need = (uint64_t)e->g.cells * capacity_per_cell;
    if (need > e->lim.max_ring_entries) {
        e->fail("chd_rings_init: %u cells x %u entries > max_ring_entries %u", e->g.cells, capacity_per_cell, e->lim.max_ring_entries);
        return CHD_ERR_CAPACITY;
    }
    CHD_ENTER(e, ENTRY_DEVICE);
    Rings& R = e->rings;
    cudaStream_t s = e->stream;
    rings_init_kernel<<<blocks_for((uint64_t)e->g.cells + 1, 128), 128, 0, s>>>(e->g.cells, capacity_per_cell, R.begin, R.end);
    KCHECK(e);
    CU(e, cudaMemsetAsync(R.set.cmi, 0, (uint64_t)e->g.cells * 8, s));
    if (R.bytes.on) CU(e, cudaMemsetAsync(R.bytes.cur, 0, 8ull * e->g.cells, s));  // empty byte slabs, the reservation kept
    set_u32_kernel<<<1, 1, 0, s>>>(R.d_total, (uint32_t)need);
    KCHECK(e);
    R.total_pending = false;
    R.owned = true;
    R.appended = R.staged;  // (a staged append is still to come: the next chd_tick_sharded applies it to these rings)
    R.after_fanout = true;
    R.cap = capacity_per_cell;
    R.view = RingDev{R.begin, R.end, R.set.arrival, R.set.sender, R.set.index, R.set.cmi, R.d_total, nullptr};
    pf_reader_reset(R);
    R.pf.staged = -1;  // host-owned rings prefetched before this call are not adopted
    return CHD_OK;
}

chd_status chd_rings_append(chd_engine* e, const uint32_t* upd_off, uint32_t n_updates, const int64_t* arrival_ns, const uint32_t* sender_conn_id) {
    if (!e || !upd_off || (n_updates && (!arrival_ns || !sender_conn_id))) return CHD_ERR_INVALID;
    if (!e->rings.owned) {
        e->fail("chd_rings_append before chd_rings_init");
        return CHD_ERR_STATE;
    }
    if (chd_rule_no_chain(e, "chd_rings_append", false) != CHD_OK || chd_rule_rings_staged(e, "chd_rings_append") != CHD_OK ||
        chd_rule_ring_append(e, false) != CHD_OK)
        return CHD_ERR_STATE;
    CHD_ENTER(e, ENTRY_DEVICE);
    return rings_append_on(e, upd_off, n_updates, arrival_ns, sender_conn_id);
}

chd_status chd_rings_apply(chd_engine* e, cudaStream_t s, uint32_t n_updates) {
    Rings& R = e->rings;
    const uint32_t C = e->g.cells;
    const Rings::RingBytes& rb = R.bytes;
    if (rb.on) {
        rings_append_bytes_kernel<<<blocks_for((uint64_t)C * 32, 128), 128, 0, s>>>(
            C, R.cap, R.upd_off, n_updates, R.upd_arrival, R.upd_sender, rb.upd_boff, rb.upd_bytes, R.begin, R.end, R.set.arrival, R.set.sender,
            R.set.index, rb.pos, rb.len, rb.slab, rb.per_cell, rb.cur, R.set.cmi, e->d_cell_max_interval, &e->d_ctr->overflow);
    } else {
        rings_append_kernel<<<blocks_for(C, 128), 128, 0, s>>>(C, R.cap, R.upd_off, n_updates, R.upd_arrival, R.upd_sender, R.begin, R.end, R.set.arrival,
                                                               R.set.sender, R.set.index, R.set.cmi, e->d_cell_max_interval, &e->d_ctr->overflow);
    }
    KCHECK(e);
    R.staged = false;
    R.after_fanout = true;
    return CHD_OK;
}

chd_status chd_get_rings(chd_engine* e, uint32_t* ring_off, int64_t* arrival_ns, uint32_t* sender_conn_id, uint64_t* message_index,
                         uint64_t* channel_msg_index, uint32_t cap_entries) {
    if (!e || !ring_off) return CHD_ERR_INVALID;
    if (!e->rings.owned) {
        e->fail("chd_get_rings: the rings are host-owned (chd_set_rings)");
        return CHD_ERR_STATE;
    }
    if (chd_rule_rings_staged(e, "chd_get_rings") != CHD_OK) return CHD_ERR_STATE;  // (its length pass reuses upd_off)
    CHD_ENTER(e, ENTRY_COPY_WAIT);
    const Rings& R = e->rings;
    cudaStream_t s = e->stream;
    const uint32_t C = e->g.cells;
    chd_status st = live_entry_csr(e);
    uint32_t total = 0;
    if (st == CHD_OK) st = chd_read_u32(e, R.flat_off + C, &total);
    if (st != CHD_OK) return st;
    CU(e, cudaMemcpyAsync(ring_off, R.flat_off, sizeof(uint32_t) * ((uint64_t)C + 1), cudaMemcpyDefault, s));
    if (channel_msg_index) CU(e, cudaMemcpyAsync(channel_msg_index, R.set.cmi, sizeof(uint64_t) * C, cudaMemcpyDefault, s));
    if (arrival_ns || sender_conn_id || message_index) {
        if (total > cap_entries) {
            e->fail("chd_get_rings: %u entries > cap_entries %u", total, cap_entries);
            return CHD_ERR_CAPACITY;
        }
        int64_t* ta = nullptr;  // (one temporary: arrival, index, sender)
        CU(e, cudaMallocAsync((void**)&ta, 20ull * (total + 1), s));
        uint64_t* ti = (uint64_t*)(ta + total + 1);
        uint32_t* ts = (uint32_t*)(ti + total + 1);
        rings_gather_kernel<<<C, 128, 0, s>>>(C, R.begin, R.end, R.flat_off, R.set.arrival, R.set.sender, R.set.index, ta, ts, ti, total);
        KCHECK(e);
        if (arrival_ns) CU(e, cudaMemcpyAsync(arrival_ns, ta, 8ull * total, cudaMemcpyDefault, s));
        if (sender_conn_id) CU(e, cudaMemcpyAsync(sender_conn_id, ts, 4ull * total, cudaMemcpyDefault, s));
        if (message_index) CU(e, cudaMemcpyAsync(message_index, ti, 8ull * total, cudaMemcpyDefault, s));
        CU(e, cudaFreeAsync(ta, s));
    }
    CU(e, cudaStreamSynchronize(s));
    return CHD_OK;
}

/* ---- byte-carrying device rings (include/chd_gpu_ring_bytes.h): each update's serialized updateMsg kept in the ring beside
   its entry (rings_append_bytes_kernel), read in place by the payload kernels (chd_payload.cuh) */

chd_status chd_rings_reserve_bytes(chd_engine* e, uint32_t bytes_per_cell) {
    if (!e) return CHD_ERR_INVALID;
    if (bytes_per_cell == 0) {
        e->fail("chd_rings_reserve_bytes: bytes_per_cell must be positive");
        return CHD_ERR_INVALID;
    }
    // (rule 12 too: staged updates were checked against the slab they were staged for, and their bytes would be applied to this one)
    if (chd_rule_ring_bytes_reserve(e) != CHD_OK || chd_rule_rings_staged(e, "chd_rings_reserve_bytes") != CHD_OK) return CHD_ERR_STATE;
    CHD_ENTER(e, ENTRY_DEVICE);
    Rings::RingBytes& rb = e->rings.bytes;
    const uint64_t C = e->g.cells;
    // a failed allocation changes nothing: the per-slot arrays are kept once made, and a new slab replaces the old one only once it exists
    const bool slots = (rb.pos || dalloc(e, &rb.pos, (uint64_t)e->lim.max_ring_entries)) && (rb.len || dalloc(e, &rb.len, (uint64_t)e->lim.max_ring_entries)) &&
                       (rb.cur || dalloc(e, &rb.cur, 2 * C));
    if (!slots) {
        cudaGetLastError();  // (an allocation failure is not sticky: clear it for the next launch check)
        return CHD_ERR_CUDA;
    }
    if (!rb.slab || rb.per_cell != bytes_per_cell) {
        uint8_t* slab = nullptr;
        if (!dalloc(e, &slab, C * bytes_per_cell)) {
            cudaGetLastError();
            e->fail("chd_rings_reserve_bytes: %llu cells x %u bytes cannot be allocated", (unsigned long long)C, bytes_per_cell);
            return CHD_ERR_CAPACITY;
        }
        chd_dfree(e, rb.slab);
        rb.slab = slab;
    }
    CU(e, cudaMemsetAsync(rb.cur, 0, 8 * C, e->stream));
    rb.per_cell = bytes_per_cell;
    rb.on = true;
    return CHD_OK;
}

chd_status chd_rings_append_bytes(chd_engine* e, const uint32_t* upd_off, uint32_t n_updates, const int64_t* arrival_ns, const uint32_t* sender_conn_id,
                                  const uint64_t* byte_off, const uint8_t* bytes) {
    if (!e || !upd_off || !byte_off || (n_updates && (!arrival_ns || !sender_conn_id))) return CHD_ERR_INVALID;
    if (!e->rings.owned) {
        e->fail("chd_rings_append_bytes before chd_rings_init");
        return CHD_ERR_STATE;
    }
    if (chd_rule_no_chain(e, "chd_rings_append_bytes", false) != CHD_OK || chd_rule_rings_staged(e, "chd_rings_append_bytes") != CHD_OK ||
        chd_rule_ring_append(e, true) != CHD_OK)
        return CHD_ERR_STATE;
    // byte_off is a host array: its lengths are checked here, before anything is appended
    for (uint32_t k = 0; k < n_updates; k++) {
        if (byte_off[k + 1] < byte_off[k] || byte_off[k + 1] - byte_off[k] > e->rings.bytes.per_cell) {
            e->fail("chd_rings_append_bytes: update %u has byte offsets %llu .. %llu (bytes_per_cell %u)", k, (unsigned long long)byte_off[k],
                    (unsigned long long)byte_off[k + 1], e->rings.bytes.per_cell);
            return CHD_ERR_INVALID;
        }
    }
    const uint64_t nb = byte_off[n_updates];
    if (nb && !bytes) {
        e->fail("chd_rings_append_bytes: %llu bytes and no byte array", (unsigned long long)nb);
        return CHD_ERR_INVALID;
    }
    CHD_ENTER(e, ENTRY_DEVICE);
    return rings_append_on(e, upd_off, n_updates, arrival_ns, sender_conn_id, byte_off, bytes);
}

chd_status chd_get_ring_bytes(chd_engine* e, uint64_t* byte_off, uint8_t* bytes, uint64_t cap_bytes, uint64_t* total) {
    if (!e) return CHD_ERR_INVALID;
    if (!e->rings.owned || !e->rings.bytes.on) {
        e->fail("chd_get_ring_bytes needs byte-carrying device rings (chd_rings_reserve_bytes)");
        return CHD_ERR_STATE;
    }
    if (chd_rule_rings_staged(e, "chd_get_ring_bytes") != CHD_OK) return CHD_ERR_STATE;  // (its length pass reuses upd_off)
    CHD_ENTER(e, ENTRY_COPY_WAIT);
    const Rings& R = e->rings;
    const Rings::RingBytes& rb = R.bytes;
    cudaStream_t s = e->stream;
    const uint32_t C = e->g.cells;
    if (total) *total = 0;
    // (control-plane call: the entry CSR as chd_get_rings makes it; the cells' byte offsets, scan scratch and lengths in one temporary)
    chd_status st = live_entry_csr(e);
    if (st != CHD_OK) return st;
    unsigned long long* cell_boff = nullptr;
    CU(e, cudaMallocAsync((void**)&cell_boff, 8ull * (C + 2 + scan_scratch_elems(C + 1)) + 4ull * C + 4, s));
    unsigned long long* scratch = cell_boff + C + 2;
    uint32_t* blen = (uint32_t*)(scratch + scan_scratch_elems(C + 1));
    ring_bytes_len_kernel<<<blocks_for(C, 128), 128, 0, s>>>(C, rb.cur, blen);
    KCHECK(e);
    SCAN(e, exclusive_scan<uint32_t, unsigned long long>(blen, cell_boff, C, scratch, s));
    uint64_t* h64 = (uint64_t*)e->h_u32;
    CU(e, cudaMemcpyAsync(h64, cell_boff + C, 8, cudaMemcpyDeviceToHost, s));
    CU(e, cudaMemcpyAsync(h64 + 1, R.flat_off + C, 4, cudaMemcpyDeviceToHost, s));
    CU(e, cudaStreamSynchronize(s));
    const uint64_t nb = h64[0];
    const uint32_t n_live = (uint32_t)h64[1];
    if (total) *total = nb;
    if (bytes && nb > cap_bytes) {
        e->fail("chd_get_ring_bytes: %llu bytes > cap_bytes %llu", (unsigned long long)nb, (unsigned long long)cap_bytes);
        st = CHD_ERR_CAPACITY;
    } else if (byte_off || bytes) {
        unsigned long long* o_boff = nullptr;  // (one temporary: entry offsets, bytes)
        CU(e, cudaMallocAsync((void**)&o_boff, 8ull * (n_live + 1) + nb + 1, s));
        uint8_t* o_bytes = (uint8_t*)(o_boff + n_live + 1);
        ring_bytes_gather_kernel<<<C, 128, 0, s>>>(C, R.begin, R.end, R.flat_off, rb.pos, rb.cur, cell_boff, rb.slab, rb.per_cell, o_boff, o_bytes);
        KCHECK(e);
        CU(e, cudaMemcpyAsync(o_boff + n_live, cell_boff + C, 8, cudaMemcpyDeviceToDevice, s));
        if (byte_off) CU(e, cudaMemcpyAsync(byte_off, o_boff, 8ull * (n_live + 1), cudaMemcpyDefault, s));
        if (bytes && nb) CU(e, cudaMemcpyAsync(bytes, o_bytes, nb, cudaMemcpyDefault, s));
        CU(e, cudaFreeAsync(o_boff, s));
    }
    CU(e, cudaFreeAsync(cell_boff, s));
    CU(e, cudaStreamSynchronize(s));
    return st;
}

}  // extern "C"
