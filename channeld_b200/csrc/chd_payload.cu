// chd_payload.cu — host side of the byte half of the fan-out (chd_payload.cuh): payload bytes in, per-class Packet entries and
// per-connection framed packets out.  Buffers of this optional stage are allocated on first use and grown on demand (not part
// of the fixed-capacity tick path).
#include "chd_engine.h"

#include "chd_payload.cuh"

#define ENSURE(e, ptr, cap, need)                                                       \
    do {                                                                                \
        const uint64_t _n = (need);                                                     \
        if (!ensure_cap(e, &(ptr), &(cap), _n, _n + _n / 4 + 256)) return CHD_ERR_CUDA; \
    } while (0)

static chd_status remake_site(chd_engine* e, ScanSite& site, uint64_t* cap, uint64_t need, int stage) {
    if (site.desc && need <= *cap) return CHD_OK;
    chd_dfree(e, site.desc);
    site.desc = nullptr;
    const uint64_t c = need + need / 4 + SCAN_TILE;
    if (!chd_make_site(e, site, c, stage)) return CHD_ERR_CUDA;
    site.error = &e->d_ctr->overflow;
    *cap = c;
    return CHD_OK;
}

extern "C" {

chd_status chd_set_payload_bytes(chd_engine* e, const uint64_t* entry_off, uint32_t n_entries, const uint8_t* entry_bytes, const uint64_t* full_off,
                                 const uint8_t* full_bytes, const char* type_url, uint32_t msg_type) {
    if (!e || !entry_off || !full_off || !type_url) return CHD_ERR_INVALID;
    if (chd_rule_payload_entries(e, n_entries) != CHD_OK) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_LOCK | ENTRY_COPY_WAIT);
    cudaStream_t s = e->stream;
    chd_engine::Payload& P = e->pl;
    const uint64_t C = e->g.cells;
    // sizes come from the last offsets (host arrays: this is a per-tick input upload like chd_set_rings)
    const uint64_t eb = entry_off[n_entries], fb = full_off[C];
    if ((eb && !entry_bytes) || (fb && !full_bytes)) return CHD_ERR_INVALID;
    const uint64_t ul = strlen(type_url);
    ENSURE(e, P.d_entry_off, P.cap_entry_off, (uint64_t)n_entries + 1);
    ENSURE(e, P.d_entry_bytes, P.cap_entry_bytes, eb + 1);
    ENSURE(e, P.d_full_off, P.cap_full_off, C + 1);
    ENSURE(e, P.d_full_bytes, P.cap_full_bytes, fb + 1);
    ENSURE(e, P.d_url, P.cap_url, ul + 1);
    CU(e, cudaMemcpyAsync(P.d_entry_off, entry_off, 8 * ((uint64_t)n_entries + 1), cudaMemcpyDefault, s));
    if (eb) CU(e, cudaMemcpyAsync(P.d_entry_bytes, entry_bytes, eb, cudaMemcpyDefault, s));
    CU(e, cudaMemcpyAsync(P.d_full_off, full_off, 8 * (C + 1), cudaMemcpyDefault, s));
    if (fb) CU(e, cudaMemcpyAsync(P.d_full_bytes, full_bytes, fb, cudaMemcpyDefault, s));
    CU(e, cudaMemcpyAsync(P.d_url, type_url, ul, cudaMemcpyHostToDevice, s));
    CU(e, cudaStreamSynchronize(s));  // type_url / host arrays may be transient
    P.url_len = (uint32_t)ul;
    P.msg_type = msg_type;
    P.n_entries = n_entries;
    P.have_input = true;
    return CHD_OK;
}

chd_status chd_assemble_payloads(chd_engine* e, uint32_t* out_n_classes, uint64_t* out_class_off, uint32_t cap_classes, uint8_t* out_blob,
                                 uint64_t blob_cap, uint64_t* out_blob_len) {
    if (!e) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_LOCK | ENTRY_COPY_WAIT);
    chd_engine::Payload& P = e->pl;
    if (!P.have_input) {
        e->fail("chd_assemble_payloads before chd_set_payload_bytes");
        return CHD_ERR_STATE;
    }
    if (chd_rule_assemble_rings(e) != CHD_OK) return CHD_ERR_STATE;
    // window classes of the last fan-out pass (results stay on the device)
    uint32_t n_classes = 0;
    chd_status st = chd_due_classes(e, nullptr, nullptr, nullptr, 0, &n_classes);
    if (st != CHD_OK) return st;
    P.n_classes = n_classes;
    if (out_n_classes) *out_n_classes = n_classes;
    if (out_blob_len) *out_blob_len = 0;
    if (n_classes == 0) {
        P.blob_len = 0;
        P.assembled = true;
        if (out_class_off && cap_classes + 1 >= 1) out_class_off[0] = 0;
        return CHD_OK;
    }
    cudaStream_t s = e->stream;
    ENSURE(e, P.d_cls_len, P.cap_cls, (uint64_t)n_classes + 1);
    ENSURE(e, P.d_cls_off, P.cap_cls_off, (uint64_t)n_classes + 2);
    st = remake_site(e, P.site_cls, &P.cap_site_cls, (uint64_t)n_classes + 1, EP_PAYLOAD);
    if (st != CHD_OK) return st;
    st = chd_ring_total_flush(e, s);
    if (st != CHD_OK) return st;
    const RingDev ring = chd_ring_view(e);
    const chd_engine::Rings::RingBytes& rb = e->rings.bytes;
    const bool dev = e->rings.owned;  // (byte-carrying: rule 14)
    const PayloadIn in{(const unsigned long long*)P.d_entry_off, P.d_entry_bytes, (const unsigned long long*)P.d_full_off, P.d_full_bytes, P.d_url, P.url_len,
                       P.msg_type, dev ? rb.slab : nullptr, dev ? rb.pos : nullptr, dev ? rb.len : nullptr, rb.per_cell};
    st = chd_epoch_tick(e, s, EP_PAYLOAD);
    if (st != CHD_OK) return st;
    payload_size_kernel<<<blocks_for(n_classes, 128), 128, 0, s>>>(n_classes, e->d_cls_out_rep, e->d_due, e->d_due_key, ring, e->d_conn, in, P.d_cls_len,
                                                                  e->d_epoch + EP_PAYLOAD);
    KCHECK(e);
    SCAN(e, exclusive_scan_1p<uint32_t, unsigned long long>(P.d_cls_len, (unsigned long long*)P.d_cls_off, n_classes, P.site_cls, s));
    uint64_t* h64 = (uint64_t*)e->h_u32;
    CU(e, cudaMemcpyAsync(h64, P.d_cls_off + n_classes, 8, cudaMemcpyDeviceToHost, s));
    CU(e, cudaStreamSynchronize(s));
    const uint64_t total = *h64;
    P.blob_len = total;
    if (out_blob_len) *out_blob_len = total;
    ENSURE(e, P.d_blob, P.cap_blob, total + 16);
    payload_write_kernel<<<blocks_for((uint64_t)n_classes * 32, 128), 128, 0, s>>>(n_classes, e->d_cls_out_rep, e->d_due, e->d_due_key, ring, e->d_conn, in,
                                                                                   (const unsigned long long*)P.d_cls_off, P.d_blob, P.cap_blob);
    KCHECK(e);
    if (out_class_off) {
        if (n_classes > cap_classes) {
            e->fail("chd_assemble_payloads: %u classes > cap_classes %u", n_classes, cap_classes);
            return CHD_ERR_CAPACITY;
        }
        CU(e, cudaMemcpyAsync(out_class_off, P.d_cls_off, 8ull * ((uint64_t)n_classes + 1), cudaMemcpyDefault, s));
    }
    if (out_blob) {
        if (total > blob_cap) {
            e->fail("chd_assemble_payloads: %llu payload bytes > blob_cap %llu", (unsigned long long)total, (unsigned long long)blob_cap);
            return CHD_ERR_CAPACITY;
        }
        CU(e, cudaMemcpyAsync(out_blob, P.d_blob, total, cudaMemcpyDefault, s));
    }
    CU(e, cudaStreamSynchronize(s));
    P.assembled = true;
    return CHD_OK;
}

chd_status chd_frame_packets(chd_engine* e, const uint8_t* compression, uint64_t* out_conn_off, uint32_t* out_conn_len, uint32_t* out_conn_frames,
                             uint8_t* out_bytes, uint64_t out_cap, uint64_t* out_len, uint32_t* out_dropped) {
    if (!e) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_LOCK | ENTRY_COPY_WAIT);
    chd_engine::Payload& P = e->pl;
    if (!P.assembled) {
        e->fail("chd_frame_packets before chd_assemble_payloads");
        return CHD_ERR_STATE;
    }
    cudaStream_t s = e->stream;
    const uint32_t S = e->n_slots;
    if (out_len) *out_len = 0;
    if (out_dropped) *out_dropped = 0;
    if (S == 0) return CHD_OK;
    uint32_t n_due = 0;
    chd_status st = chd_read_u32(e, &e->d_ctr->n_due, &n_due);
    if (st != CHD_OK) return st;
    if (n_due > e->lim.max_due) n_due = e->lim.max_due;
    ENSURE(e, P.d_fc_cnt, P.cap_fc, (uint64_t)S + 2);
    ENSURE(e, P.d_fc_off, P.cap_fc_off, (uint64_t)S + 2);
    ENSURE(e, P.d_fc_cursor, P.cap_fc_cur, (uint64_t)S + 2);
    ENSURE(e, P.d_fc_idx, P.cap_fc_idx, (uint64_t)e->lim.max_due + 1);
    ENSURE(e, P.d_conn_cap, P.cap_conn_cap, (uint64_t)S + 2);
    ENSURE(e, P.d_conn_off, P.cap_conn_off, (uint64_t)S + 2);
    ENSURE(e, P.d_conn_len, P.cap_conn_len, (uint64_t)S + 2);
    ENSURE(e, P.d_conn_frames, P.cap_conn_frames, (uint64_t)S + 2);
    ENSURE(e, P.d_comp, P.cap_comp, (uint64_t)S + 2);
    ENSURE(e, P.d_ndrop, P.cap_ndrop, 2);
    st = remake_site(e, P.site_fc, &P.cap_site_fc, (uint64_t)S + 1, EP_PAYLOAD);
    if (st != CHD_OK) return st;
    st = remake_site(e, P.site_conn, &P.cap_site_conn, (uint64_t)S + 1, EP_PAYLOAD);
    if (st != CHD_OK) return st;
    CU(e, cudaMemsetAsync(P.d_fc_cnt, 0, 4ull * (S + 1), s));
    CU(e, cudaMemsetAsync(P.d_fc_cursor, 0, 4ull * (S + 1), s));
    CU(e, cudaMemsetAsync(P.d_ndrop, 0, 4, s));
    if (compression) CU(e, cudaMemcpyAsync(P.d_comp, compression, S, cudaMemcpyDefault, s));
    st = chd_epoch_tick(e, s, EP_PAYLOAD);
    if (st != CHD_OK) return st;
    frame_count_kernel<<<blocks_for(n_due ? n_due : 1, 256), 256, 0, s>>>(e->d_due, n_due, S, P.d_fc_cnt, e->d_epoch + EP_PAYLOAD);
    KCHECK(e);
    SCAN(e, exclusive_scan_1p<uint32_t, uint32_t>(P.d_fc_cnt, P.d_fc_off, S, P.site_fc, s));
    if (n_due) {
        frame_fill_kernel<<<blocks_for(n_due, 256), 256, 0, s>>>(e->d_due, n_due, S, P.d_fc_off, P.d_fc_cursor, P.d_fc_idx);
        KCHECK(e);
    }
    frame_size_kernel<<<blocks_for(S, 128), 128, 0, s>>>(S, P.d_fc_off, P.d_fc_idx, e->d_cls_of, P.d_cls_len, compression ? P.d_comp : nullptr, P.d_conn_cap,
                                                        P.d_ndrop);
    KCHECK(e);
    SCAN(e, exclusive_scan_1p<uint32_t, unsigned long long>(P.d_conn_cap, (unsigned long long*)P.d_conn_off, S, P.site_conn, s));
    uint64_t* h64 = (uint64_t*)e->h_u32;
    CU(e, cudaMemcpyAsync(h64, P.d_conn_off + S, 8, cudaMemcpyDeviceToHost, s));
    CU(e, cudaMemcpyAsync(h64 + 1, P.d_ndrop, 4, cudaMemcpyDeviceToHost, s));
    CU(e, cudaStreamSynchronize(s));
    const uint64_t total = h64[0];
    if (out_dropped) *out_dropped = (uint32_t)h64[1];
    if (out_len) *out_len = total;
    ENSURE(e, P.d_out, P.cap_out, total + 16);
    if (compression) ENSURE(e, P.d_stage, P.cap_stage, total + 16);
    frame_write_kernel<<<blocks_for((uint64_t)S * 32, 128), 128, 0, s>>>(S, P.d_fc_off, P.d_fc_idx, e->d_cls_of, P.d_cls_len, (const unsigned long long*)P.d_cls_off,
                                                                        P.d_blob, compression ? P.d_comp : nullptr, (const unsigned long long*)P.d_conn_off,
                                                                        P.d_out, P.cap_out, compression ? P.d_stage : P.d_out, P.d_conn_len, P.d_conn_frames);
    KCHECK(e);
    if (out_conn_off) CU(e, cudaMemcpyAsync(out_conn_off, P.d_conn_off, 8ull * (S + 1), cudaMemcpyDefault, s));
    if (out_conn_len) CU(e, cudaMemcpyAsync(out_conn_len, P.d_conn_len, 4ull * S, cudaMemcpyDefault, s));
    if (out_conn_frames) CU(e, cudaMemcpyAsync(out_conn_frames, P.d_conn_frames, 4ull * S, cudaMemcpyDefault, s));
    if (out_bytes) {
        if (total > out_cap) {
            e->fail("chd_frame_packets: %llu bytes > out_cap %llu", (unsigned long long)total, (unsigned long long)out_cap);
            return CHD_ERR_CAPACITY;
        }
        CU(e, cudaMemcpyAsync(out_bytes, P.d_out, total, cudaMemcpyDefault, s));
    }
    CU(e, cudaStreamSynchronize(s));
    return CHD_OK;
}

}  // extern "C"
