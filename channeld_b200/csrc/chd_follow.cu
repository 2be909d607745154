// chd_follow.cu — followers: subscriber slots bound to an entity and an AOI shape, and the tick's query batch generated from the
// bindings on the device (chd_follow.cuh).
//
// One generated batch is enough (chd_prefetch_queries needs two staging sets because its uploads run on another stream while a
// tick is in flight): the generation runs on the engine stream, and the interest update that reads the batch is either on the
// engine stream too or on the second stream between the tick's fork and its join, which the engine stream waits for before the
// tick ends.  A generation enqueued after that tick is therefore ordered after the last read of the batch; while a
// chd_begin_interest is pending (forked, not joined yet) chd_follow_queries is refused.  A merged generation
// (chd_follow_queries_with) also reads the host part, from the query scratch or an adopted prefetch set, on the same stream; it
// copies everything into follower-owned arrays, so the prefetch set is released right after it.
#include "chd_engine.h"

#include "chd_follow.cuh"
#include "chd_gpu_facing.h"
#include "chd_misc.cuh"

namespace {

constexpr uint32_t SHAPE_KINDS = CHD_AOI_SPHERE | CHD_AOI_BOX | CHD_AOI_CONE;

bool follow_alloc(chd_engine* e) {
    chd_engine::Follow& F = e->fw;
    if (F.on) return true;
    const uint64_t S = e->lim.max_subscribers, Q = e->lim.max_queries;
    FollowDev& d = F.st;
    FollowBatch& q = F.q;
    bool ok = dalloc(e, &d.entity, S) && dalloc(e, &d.kind, S) && dalloc(e, &d.dirty, S) && dalloc(e, &d.tslot, S) && dalloc(e, &d.res, S) &&
              dalloc(e, &d.ovr, S);
    for (double** p : {&d.sph_r, &d.box_ex, &d.box_ez, &d.cone_dx, &d.cone_dz, &d.cone_angle, &d.cone_r, &d.last_x, &d.last_z}) ok = ok && dalloc(e, p, S);
    ok = ok && dalloc(e, &q.sub, Q) && dalloc(e, &q.kind, Q) && dalloc(e, &q.n_selected, 1) && dalloc(e, &q.spot_off, Q + 1) &&
         dalloc(e, &q.spot_ndist, Q) && dalloc(e, &q.missing, Q) && dalloc(e, &F.hdr, 1);
    for (double** p : {&q.sph_cx, &q.sph_cz, &q.sph_r, &q.box_cx, &q.box_cz, &q.box_ex, &q.box_ez, &q.cone_cx, &q.cone_cz, &q.cone_dx, &q.cone_dz,
                       &q.cone_angle, &q.cone_r})
        ok = ok && dalloc(e, p, Q);
    ok = ok && chd_make_site(e, F.site, S + 1, EP_FOLLOW);
    if (!ok) return false;
    if (cudaMemsetAsync(d.kind, 0, S, e->stream) != cudaSuccess || cudaMemsetAsync(d.ovr, 0, S, e->stream) != cudaSuccess ||
        cudaMemsetAsync(q.n_selected, 0, 4, e->stream) != cudaSuccess)
        return e->fail("cudaMemsetAsync failed allocating the follower state");
    F.h_kind.assign(S, 0);
    F.on = true;
    return true;
}

// The frame state, at the first chd_follow_set_frame: no slot has a frame yet.
bool frame_alloc(chd_engine* e) {
    chd_engine::Follow& F = e->fw;
    if (F.fr.on) return true;
    const uint64_t S = e->lim.max_subscribers;
    FollowFrame d{};
    bool ok = dalloc(e, &d.on, S);
    for (double** p : {&d.off_fwd, &d.off_right, &d.rot_cos, &d.rot_sin, &d.last_fx, &d.last_fz, &d.cx, &d.cz, &d.dx, &d.dz}) ok = ok && dalloc(e, p, S);
    if (!ok) return false;
    if (cudaMemsetAsync(d.on, 0, S, e->stream) != cudaSuccess) return e->fail("cudaMemsetAsync failed allocating the frame state");
    F.h_frame.assign(S, 0);
    F.fr = d;
    return true;
}

// The slot's follower is plain again (its device mark is cleared by the caller's kernel)
void frame_forget(chd_engine::Follow& F, uint32_t s) {
    if (F.h_frame.empty() || !F.h_frame[s]) return;
    F.h_frame[s] = 0;
    F.n_framed--;
}

// The follow compaction of the generation: the instantiation for the engine's state (served-range check, frames)
template <bool Merged>
chd_status follow_compact(chd_engine* e, cudaStream_t s, bool check, bool frame, const FollowEntities& ent, const FollowSlab& slab, uint32_t mode,
                          uint32_t base) {
    chd_engine::Follow& F = e->fw;
    const uint32_t S = e->n_slots;
    if (frame && check)
        SCAN(e, compact_1p(FollowFlag<Merged, true, true>{F.st, ent, slab, mode, F.fr}, FollowSink<Merged, true>{F.st, F.q, base, F.fr}, S, F.site, s));
    else if (frame)
        SCAN(e, compact_1p(FollowFlag<Merged, false, true>{F.st, ent, slab, mode, F.fr}, FollowSink<Merged, true>{F.st, F.q, base, F.fr}, S, F.site, s));
    else if (check)
        SCAN(e, compact_1p(FollowFlag<Merged, true>{F.st, ent, slab, mode}, FollowSink<Merged>{F.st, F.q, base}, S, F.site, s));
    else
        SCAN(e, compact_1p(FollowFlag<Merged, false>{F.st, ent, slab, mode}, FollowSink<Merged>{F.st, F.q, base}, S, F.site, s));
    return CHD_OK;
}

// `bytes` of host data into the follower staging buffer, before the call returns (the caller's arrays are plain host memory)
chd_status stage_upload(chd_engine* e, const void* h, uint64_t bytes) {
    chd_engine::Follow& F = e->fw;
    if (!ensure_cap(e, &F.d_stage, &F.stage_cap, bytes, bytes + bytes / 2 + 4096)) return CHD_ERR_CUDA;
    CU(e, cudaMemcpyAsync(F.d_stage, h, bytes, cudaMemcpyHostToDevice, e->stream));
    CU(e, cudaStreamSynchronize(e->stream));
    return CHD_OK;
}

// The size class of a merged batch's host part: 0, or max(256, the next power of two >= n)
uint64_t host_class(uint32_t n) {
    if (!n) return 0;
    uint64_t H = 256;
    while (H < n) H <<= 1;
    return H;
}

// Merged batches: room for `spots` spots (at least one, so that the spot arrays exist whenever the host part has spot_off).  The
// arrays are replaced, not kept: the merge rewrites them before anything reads them.
bool spot_alloc(chd_engine* e, uint64_t spots) {
    chd_engine::Follow& F = e->fw;
    const uint64_t need = std::max<uint64_t>(spots, 1), cap = std::max<uint64_t>(need + need / 2, 4096);
    if (need <= F.spot_cap) return true;
    if (!ensure_cap(e, &F.spot_buf, &F.spot_bytes, 20 * need, 20 * cap)) return false;
    F.spot_cap = cap;
    F.q.spot_x = reinterpret_cast<double*>(F.spot_buf);
    F.q.spot_z = F.q.spot_x + cap;
    F.q.spot_dist = reinterpret_cast<uint32_t*>(F.q.spot_z + cap);
    return true;
}

// The follow stage on the engine stream: the batch generated from the bindings, behind the host part h of n_h entries (spots: its
// spot total) when n_h > 0.
chd_status follow_generate(chd_engine* e, uint32_t mode, const QueryDev& h, uint32_t n_h, uint32_t spots) {
    chd_engine::Follow& F = e->fw;
    const bool merged = n_h > 0;
    if (!merged && (!F.on || !F.n_bound)) {  // nothing follows: an empty batch (it still applies pending lifecycle changes)
        F.view = QueryDev{};
        F.ready = true;
        return CHD_OK;
    }
    cudaStream_t s = e->stream;
    StageTimer timer(e, s, CHD_STAGE_FOLLOW);
    const uint32_t S = e->n_slots, B = F.n_bound, H = (uint32_t)host_class(n_h);
    const Positions p = chd_positions(e);  // (entity-table mode: the front pair)
    const FollowEntities ent = e->tbl.on ? FollowEntities{p.x, p.z, e->lim.max_entities, e->tbl.d_table, e->tbl.bits, e->tbl.d_id_of_slot, e->tbl.d_fx, e->tbl.d_fz}
                                         : FollowEntities{p.x, p.z, e->n_own, nullptr, 0, nullptr, nullptr, nullptr};
    const bool frame = F.n_framed > 0;  // (entity-table mode only, rule 11)
    // on a slab (entity-table mode: every followed entity is an own one) the columns it serves, with the world's edges left open
    const uint32_t lo = e->slab && e->g.col_lo > e->g.halo ? e->g.col_lo - e->g.halo : 0u;
    const uint32_t hi = e->slab ? (uint32_t)std::min<uint64_t>((uint64_t)e->g.col_hi + e->g.halo, e->g.cols) : e->g.cols;
    const FollowSlab slab{e->g.off_x, e->g.w, (double)e->g.cols, lo > 0 ? (double)lo : -INFINITY, hi < e->g.cols ? (double)hi : INFINITY};
    const bool check = lo > 0 || hi < e->g.cols;
    chd_status st = chd_epoch_tick(e, s, EP_FOLLOW);
    if (st != CHD_OK) return st;
    const FollowBatch& q = F.q;
    if (!merged) {
        // the graph bakes in the slot and follower counts, the mode, where the positions and facings live (the state arrays never
        // move), the served columns and whether frames run
        const uint64_t key = stage_key(0x666f6c6cull, S, B, mode, ent.px, ent.pz, ent.n, ent.table, ent.bits, F.st.kind, q.sub, lo, hi, frame, ent.fx,
                                       F.fr.on);
        st = run_stage(e, s, F.g, key, [&]() -> chd_status {
            // the skip tail: entries behind the selected count name no slot and no kind
            CU(e, cudaMemsetAsync(q.sub, 0xFF, 4ull * B, s));
            CU(e, cudaMemsetAsync(q.kind, 0, B, s));
            bump_epoch_kernel<<<1, 1, 0, s>>>(e->d_epoch + EP_FOLLOW);
            KCHECK(e);
            return follow_compact<false>(e, s, check, frame, ent, slab, mode, 0);
        });
    } else {
        if (h.spot_off && !spot_alloc(e, spots)) return CHD_ERR_CUDA;
        // the host count changes from tick to tick inside one size class: it is read from F.hdr, not baked into the graph
        set_u32_kernel<<<1, 1, 0, s>>>(F.hdr, n_h);
        KCHECK(e);
        FollowMerge m{h, F.hdr, H, H + B, S, q, F.st.ovr};
        m.h.n = 0;
        const unsigned grid = (unsigned)std::min<uint64_t>(blocks_for(std::max<uint64_t>(H + B + 1ull, F.spot_cap), FOLLOW_THREADS), 4ull * e->sm_count);
        // ... and so do the host part's arrays (the staging set of the query scratch or a prefetch, or the caller's device arrays) and
        // the spot buffer's three arrays: a grown buffer may start where the old one did, but its spot_z and spot_dist move with the
        // capacity
        const uint64_t key = stage_key(0x666f6c6dull, S, B, H, mode, ent.px, ent.pz, ent.n, ent.table, ent.bits, F.st.kind, q.sub, lo, hi, frame, ent.fx,
                                       F.fr.on, grid, h.sub, h.kind,
                                       h.sph_cx, h.sph_cz, h.sph_r, h.box_cx, h.box_cz, h.box_ex, h.box_ez, h.cone_cx, h.cone_cz, h.cone_dx, h.cone_dz,
                                       h.cone_angle, h.cone_r, h.spot_off, h.spot_ndist, h.spot_x, h.spot_z, h.spot_dist, q.spot_x, q.spot_z,
                                       q.spot_dist, F.spot_cap);
        st = run_stage(e, s, F.g, key, [&]() -> chd_status {
            bump_epoch_kernel<<<1, 1, 0, s>>>(e->d_epoch + EP_FOLLOW);
            KCHECK(e);
            follow_merge_kernel<<<grid, FOLLOW_THREADS, 0, s>>>(m);
            KCHECK(e);
            return follow_compact<true>(e, s, check, frame, ent, slab, mode, H);
        });
    }
    if (st != CHD_OK) return st;
    if (!e->tbl.on) {  // the positions were read: a prefetch may refill their buffers after this
        st = chd_note_pos_read(e, s);
        if (st != CHD_OK) return st;
    }
    QueryDev v{};
    v.n = H + B;
    v.sub = q.sub; v.kind = q.kind;
    v.sph_cx = q.sph_cx; v.sph_cz = q.sph_cz; v.sph_r = q.sph_r;
    v.box_cx = q.box_cx; v.box_cz = q.box_cz; v.box_ex = q.box_ex; v.box_ez = q.box_ez;
    v.cone_cx = q.cone_cx; v.cone_cz = q.cone_cz; v.cone_dx = q.cone_dx; v.cone_dz = q.cone_dz; v.cone_angle = q.cone_angle; v.cone_r = q.cone_r;
    if (merged) {
        v.missing = q.missing;
        if (h.spot_off) {
            v.spot_off = q.spot_off; v.spot_ndist = q.spot_ndist; v.spot_x = q.spot_x; v.spot_z = q.spot_z; v.spot_dist = q.spot_dist;
        }
    }
    F.view = v;
    F.ready = true;
    return CHD_OK;
}

}  // namespace

extern "C" {

chd_status chd_follow_bind(chd_engine* e, const chd_follow_batch* b) {
    if (!e || !b || (b->n && (!b->slot || !b->entity))) return CHD_ERR_INVALID;
    if (chd_rule_follow(e, "chd_follow_bind") != CHD_OK) return CHD_ERR_STATE;
    const uint32_t n = b->n;
    if (!n) return CHD_OK;
    CHD_ENTER(e, ENTRY_LOCK | ENTRY_DEVICE);
    // argument checks first: a refused call binds nothing
    std::unordered_map<uint32_t, uint32_t> last;  // slot -> its last binding in the call
    last.reserve(n);
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t s = b->slot[i], kind = b->kind ? b->kind[i] : (uint32_t)CHD_AOI_SPHERE;
        if (s >= e->lim.max_subscribers || s >= e->n_slots) {
            e->fail("chd_follow_bind: slot %u was never added (%u slots, max_subscribers %u)", s, e->n_slots, e->lim.max_subscribers);
            return CHD_ERR_INVALID;
        }
        if (kind & CHD_AOI_SPOTS) {
            e->fail("chd_follow_bind: CHD_AOI_SPOTS has absolute positions and cannot follow an entity (binding %u)", i);
            return CHD_ERR_INVALID;
        }
        if (!kind || (kind & ~SHAPE_KINDS)) {
            e->fail("chd_follow_bind: kind 0x%x of binding %u is not a mask of CHD_AOI_SPHERE | CHD_AOI_BOX | CHD_AOI_CONE", kind, i);
            return CHD_ERR_INVALID;
        }
        if (((kind & CHD_AOI_SPHERE) && !b->sph_r) || ((kind & CHD_AOI_BOX) && (!b->box_ex || !b->box_ez)) ||
            ((kind & CHD_AOI_CONE) && (!b->cone_dx || !b->cone_dz || !b->cone_angle || !b->cone_r))) {
            e->fail("chd_follow_bind: binding %u has kind 0x%x but a shape array of that kind is NULL", i, kind);
            return CHD_ERR_INVALID;
        }
        last[s] = i;
    }
    chd_engine::Follow& F = e->fw;
    uint64_t fresh = 0;
    for (const auto& kv : last) fresh += !(F.on && F.h_kind[kv.first]);
    if (F.n_bound + fresh > e->lim.max_queries) {
        e->fail("chd_follow_bind: %llu followers > max_queries %u", (unsigned long long)(F.n_bound + fresh), e->lim.max_queries);
        return CHD_ERR_CAPACITY;
    }
    if (!follow_alloc(e)) return CHD_ERR_CUDA;
    // staged SoA of the m winners: shape [7][m] doubles | slot [m] | entity [m] | kind [m]
    const uint64_t m = last.size();
    std::vector<uint8_t> h(m * (7 * 8 + 4 + 4 + 1));
    double* shape = reinterpret_cast<double*>(h.data());
    uint32_t* hs = reinterpret_cast<uint32_t*>(h.data() + 56 * m);
    uint32_t* he = hs + m;
    uint8_t* hk = reinterpret_cast<uint8_t*>(he + m);
    const double* src[7] = {b->sph_r, b->box_ex, b->box_ez, b->cone_dx, b->cone_dz, b->cone_angle, b->cone_r};
    uint64_t j = 0;
    for (uint32_t i = 0; i < n; i++) {
        if (last[b->slot[i]] != i) continue;
        hs[j] = b->slot[i];
        he[j] = b->entity[i];
        hk[j] = b->kind ? b->kind[i] : (uint8_t)CHD_AOI_SPHERE;
        for (int a = 0; a < 7; a++) shape[a * m + j] = src[a] ? src[a][i] : 0.0;
        j++;
    }
    chd_status st = stage_upload(e, h.data(), h.size());
    if (st != CHD_OK) return st;
    const uint8_t* d = F.d_stage;
    const FollowStage stage{reinterpret_cast<const uint32_t*>(d + 56 * m), reinterpret_cast<const uint32_t*>(d + 60 * m), d + 64 * m,
                            reinterpret_cast<const double*>(d)};
    follow_bind_kernel<<<blocks_for(m, FOLLOW_THREADS), FOLLOW_THREADS, 0, e->stream>>>(stage, (uint32_t)m, F.st, F.fr.on);
    KCHECK(e);
    for (uint64_t k = 0; k < m; k++) {
        F.n_bound += !F.h_kind[hs[k]];
        F.h_kind[hs[k]] = hk[k];
        frame_forget(F, hs[k]);
    }
    return CHD_OK;
}

chd_status chd_follow_drop(chd_engine* e, const uint32_t* slot, const uint32_t* d_slot, uint32_t n) {
    chd_engine::Follow& F = e->fw;
    if (!F.on || !F.n_bound) return CHD_OK;
    const uint32_t S = e->lim.max_subscribers;
    if (!slot) {  // every slot
        CU(e, cudaMemsetAsync(F.st.kind, 0, S, e->stream));
        if (F.fr.on) CU(e, cudaMemsetAsync(F.fr.on, 0, S, e->stream));
        std::fill(F.h_kind.begin(), F.h_kind.end(), (uint8_t)0);
        std::fill(F.h_frame.begin(), F.h_frame.end(), (uint8_t)0);
        F.n_bound = 0;
        F.n_framed = 0;
        return CHD_OK;
    }
    uint32_t hit = 0;
    for (uint32_t i = 0; i < n; i++)
        if (slot[i] < S && F.h_kind[slot[i]]) {
            F.h_kind[slot[i]] = 0;
            frame_forget(F, slot[i]);
            hit++;
        }
    if (!hit) return CHD_OK;
    F.n_bound -= hit;
    if (!d_slot) {
        chd_status st = stage_upload(e, slot, 4ull * n);
        if (st != CHD_OK) return st;
        d_slot = reinterpret_cast<const uint32_t*>(F.d_stage);
    }
    follow_unbind_kernel<<<blocks_for(n, FOLLOW_THREADS), FOLLOW_THREADS, 0, e->stream>>>(d_slot, n, S, F.st.kind, F.fr.on);
    KCHECK(e);
    return CHD_OK;
}

chd_status chd_follow_unbind(chd_engine* e, const uint32_t* slot, uint32_t n) {
    if (!e || (n && !slot)) return CHD_ERR_INVALID;
    if (chd_rule_follow(e, "chd_follow_unbind") != CHD_OK) return CHD_ERR_STATE;
    if (!n) return CHD_OK;
    CHD_ENTER(e, ENTRY_LOCK | ENTRY_DEVICE);
    for (uint32_t i = 0; i < n; i++)
        if (slot[i] >= e->lim.max_subscribers) {
            e->fail("chd_follow_unbind: slot %u >= max_subscribers %u", slot[i], e->lim.max_subscribers);
            return CHD_ERR_INVALID;
        }
    return chd_follow_drop(e, slot, nullptr, n);
}

chd_status chd_follow_queries(chd_engine* e, uint32_t mode) {
    if (!e || (mode != CHD_FOLLOW_ALL && mode != CHD_FOLLOW_MOVED)) return CHD_ERR_INVALID;
    if (chd_rule_follow(e, "chd_follow_queries") != CHD_OK || chd_rule_one_batch(e, "chd_follow_queries") != CHD_OK) return CHD_ERR_STATE;
    CHD_ENTER(e, ENTRY_LOCK | ENTRY_DEVICE);
    return follow_generate(e, mode, QueryDev{}, 0, 0);
}

chd_status chd_follow_queries_with(chd_engine* e, uint32_t mode, const chd_query_batch* q) {
    if (!e || (mode != CHD_FOLLOW_ALL && mode != CHD_FOLLOW_MOVED)) return CHD_ERR_INVALID;
    if (chd_rule_follow(e, "chd_follow_queries_with") != CHD_OK || chd_rule_merged_batch(e, !q) != CHD_OK) return CHD_ERR_STATE;
    CHD_ENTER(e, ENTRY_LOCK | ENTRY_DEVICE);
    chd_engine::Follow& F = e->fw;
    const int set = q ? -1 : e->pf_q.cur;  // the adopted prefetch set holding the host part
    const QueryDev* adopted = q ? nullptr : &e->dq_pf[set].view;
    if (q ? !q->sub : !adopted->sub) {
        e->fail("chd_follow_queries_with: the host part is an identity batch (sub == NULL), which cannot be merged");
        return CHD_ERR_INVALID;
    }
    const uint32_t n_h = q ? q->n : adopted->n;
    const uint64_t len = host_class(n_h) + (F.on ? F.n_bound : 0);
    if (len > e->lim.max_queries) {
        e->fail("chd_follow_queries_with: merged batch of %llu entries (%u host entries in a class of %llu, %u followers) > max_queries %u",
                (unsigned long long)len, n_h, (unsigned long long)host_class(n_h), F.n_bound, e->lim.max_queries);
        return CHD_ERR_CAPACITY;
    }
    QueryDev h{};
    uint32_t spots = 0;
    chd_status st = CHD_OK;
    if (n_h && q) {
        st = chd_upload_queries(e, e->stream, q, &h, true, nullptr, &spots);  // into the query scratch, which the merge reads on the same stream
    } else if (adopted) {  // ordered after the upload like any reader of an adopted set, whether or not the part is empty
        h = *adopted;
        spots = e->dq_pf[set].spots;
        st = chd_pf_wait(e, e->pf_q, e->stream);
    }
    if (st != CHD_OK) return st;
    if (n_h && !follow_alloc(e)) return CHD_ERR_CUDA;
    st = follow_generate(e, mode, h, n_h, spots);
    if (st != CHD_OK || set < 0) return st;
    e->pf_q.cur = -1;  // consumed: the staging set may be refilled once the merge has read it
    return chd_pf_note_read(e, e->pf_q, set, e->stream);
}

chd_status chd_get_follow(chd_engine* e, uint32_t* slot, uint32_t* entity, uint32_t* status, double* cx, double* cz, uint32_t cap, uint32_t* count,
                          uint32_t* n_selected) {
    if (!e) return CHD_ERR_INVALID;
    if (chd_rule_follow(e, "chd_get_follow") != CHD_OK) return CHD_ERR_STATE;
    if (chd_rule_no_generated_batch(e, "chd_get_follow") != CHD_OK || chd_rule_no_chain(e, "chd_get_follow", false) != CHD_OK) return CHD_ERR_STATE;
    chd_engine::Follow& F = e->fw;
    if (count) *count = 0;
    if (n_selected) *n_selected = 0;
    if (!F.on || !F.n_bound) return CHD_OK;
    CHD_ENTER(e, ENTRY_LOCK | ENTRY_COPY_WAIT);
    cudaStream_t s = e->stream;
    const uint64_t Q = e->lim.max_queries;
    if (!F.g_count && !(dalloc(e, &F.g_slot, Q) && dalloc(e, &F.g_entity, Q) && dalloc(e, &F.g_status, Q) && dalloc(e, &F.g_cx, Q) && dalloc(e, &F.g_cz, Q) &&
                        dalloc(e, &F.g_count, 1)))
        return CHD_ERR_CUDA;  // (g_count is allocated last)
    chd_status st = chd_epoch_tick(e, s, EP_FOLLOW);
    if (st != CHD_OK) return st;
    bump_epoch_kernel<<<1, 1, 0, s>>>(e->d_epoch + EP_FOLLOW);
    KCHECK(e);
    SCAN(e, compact_1p(FollowBoundFlag{F.st.kind}, FollowReportSink{F.st, e->d_status, F.g_slot, F.g_entity, F.g_status, F.g_cx, F.g_cz, F.g_count}, e->n_slots,
                       F.site, s));
    uint32_t m = 0;
    st = chd_read_u32(e, F.g_count, &m);
    if (st != CHD_OK) return st;
    if (count) *count = m;
    if (n_selected) {
        st = chd_read_u32(e, F.q.n_selected, n_selected);
        if (st != CHD_OK) return st;
    }
    const uint64_t k = std::min(m, cap);
    if (!k) return CHD_OK;
    if (slot) CU(e, cudaMemcpyAsync(slot, F.g_slot, 4 * k, cudaMemcpyDefault, s));
    if (entity) CU(e, cudaMemcpyAsync(entity, F.g_entity, 4 * k, cudaMemcpyDefault, s));
    if (status) CU(e, cudaMemcpyAsync(status, F.g_status, 4 * k, cudaMemcpyDefault, s));
    if (cx) CU(e, cudaMemcpyAsync(cx, F.g_cx, 8 * k, cudaMemcpyDefault, s));
    if (cz) CU(e, cudaMemcpyAsync(cz, F.g_cz, 8 * k, cudaMemcpyDefault, s));
    CU(e, cudaStreamSynchronize(s));
    return CHD_OK;
}

// ---- frames (include/chd_gpu_facing.h)

chd_status chd_follow_set_frame(chd_engine* e, const chd_follow_frame_batch* b) {
    if (!e || !b || (b->n && !b->slot) || (!b->rot_cos != !b->rot_sin)) return CHD_ERR_INVALID;
    if (chd_rule_facing(e, "chd_follow_set_frame") != CHD_OK || chd_rule_follow(e, "chd_follow_set_frame") != CHD_OK) return CHD_ERR_STATE;
    const uint32_t n = b->n;
    if (!n) return CHD_OK;
    CHD_ENTER(e, ENTRY_LOCK | ENTRY_DEVICE);
    chd_engine::Follow& F = e->fw;
    // argument checks first: a refused call frames nothing
    std::unordered_map<uint32_t, uint32_t> last;  // slot -> its last frame in the call
    last.reserve(n);
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t s = b->slot[i];
        if (!F.on || s >= e->lim.max_subscribers || !F.h_kind[s]) {
            e->fail("chd_follow_set_frame: slot %u follows nothing (chd_follow_bind first)", s);
            return CHD_ERR_INVALID;
        }
        const double v[4] = {b->off_fwd ? b->off_fwd[i] : 0.0, b->off_right ? b->off_right[i] : 0.0, b->rot_cos ? b->rot_cos[i] : 1.0,
                             b->rot_sin ? b->rot_sin[i] : 0.0};
        for (double a : v)
            if (!std::isfinite(a)) {
                e->fail("chd_follow_set_frame: frame %u (slot %u) has a non-finite offset or rotation", i, s);
                return CHD_ERR_INVALID;
            }
        last[s] = i;
    }
    if (!frame_alloc(e)) return CHD_ERR_CUDA;
    // staged SoA of the m winners: [4][m] doubles (off_fwd, off_right, rot_cos, rot_sin) | slot [m]
    const uint64_t m = last.size();
    std::vector<uint8_t> h(m * (4 * 8 + 4));
    double* v = reinterpret_cast<double*>(h.data());
    uint32_t* hs = reinterpret_cast<uint32_t*>(h.data() + 32 * m);
    uint64_t j = 0;
    for (uint32_t i = 0; i < n; i++) {
        if (last[b->slot[i]] != i) continue;
        hs[j] = b->slot[i];
        v[j] = b->off_fwd ? b->off_fwd[i] : 0.0;
        v[m + j] = b->off_right ? b->off_right[i] : 0.0;
        v[2 * m + j] = b->rot_cos ? b->rot_cos[i] : 1.0;
        v[3 * m + j] = b->rot_sin ? b->rot_sin[i] : 0.0;
        j++;
    }
    chd_status st = stage_upload(e, h.data(), h.size());
    if (st != CHD_OK) return st;
    const FollowFrameStage stage{reinterpret_cast<const uint32_t*>(F.d_stage + 32 * m), reinterpret_cast<const double*>(F.d_stage)};
    follow_frame_kernel<<<blocks_for(m, FOLLOW_THREADS), FOLLOW_THREADS, 0, e->stream>>>(stage, (uint32_t)m, F.st, F.fr);
    KCHECK(e);
    for (uint64_t k = 0; k < m; k++) {
        F.n_framed += !F.h_frame[hs[k]];
        F.h_frame[hs[k]] = 1;
    }
    return CHD_OK;
}

chd_status chd_get_follow_frame(chd_engine* e, uint32_t* slot, double* fx, double* fz, double* cx, double* cz, double* dx, double* dz, uint32_t cap,
                                uint32_t* count) {
    if (!e) return CHD_ERR_INVALID;
    if (chd_rule_facing(e, "chd_get_follow_frame") != CHD_OK || chd_rule_follow(e, "chd_get_follow_frame") != CHD_OK) return CHD_ERR_STATE;
    if (chd_rule_no_generated_batch(e, "chd_get_follow_frame") != CHD_OK || chd_rule_no_chain(e, "chd_get_follow_frame", false) != CHD_OK)
        return CHD_ERR_STATE;
    chd_engine::Follow& F = e->fw;
    if (count) *count = 0;
    if (!F.on || !F.n_framed) return CHD_OK;
    CHD_ENTER(e, ENTRY_LOCK | ENTRY_COPY_WAIT);
    cudaStream_t s = e->stream;
    const uint64_t Q = e->lim.max_queries;
    if (!F.g_fval && !(dalloc(e, &F.g_fslot, Q + 1) && dalloc(e, &F.g_fval, 6 * Q))) return CHD_ERR_CUDA;  // (g_fval is allocated last)
    uint32_t* d_count = F.g_fslot + Q;
    chd_status st = chd_epoch_tick(e, s, EP_FOLLOW);
    if (st != CHD_OK) return st;
    bump_epoch_kernel<<<1, 1, 0, s>>>(e->d_epoch + EP_FOLLOW);
    KCHECK(e);
    SCAN(e, compact_1p(FollowFramedFlag{F.st.kind, F.fr.on}, FollowFrameReportSink{F.fr, F.g_fslot, F.g_fval, (uint32_t)Q, d_count}, e->n_slots, F.site, s));
    uint32_t m = 0;
    st = chd_read_u32(e, d_count, &m);
    if (st != CHD_OK) return st;
    if (count) *count = m;
    const uint64_t k = std::min(m, cap);
    if (!k) return CHD_OK;
    if (slot) CU(e, cudaMemcpyAsync(slot, F.g_fslot, 4 * k, cudaMemcpyDefault, s));
    double* out[6] = {fx, fz, cx, cz, dx, dz};
    for (int a = 0; a < 6; a++)
        if (out[a]) CU(e, cudaMemcpyAsync(out[a], F.g_fval + a * Q, 8 * k, cudaMemcpyDefault, s));
    CU(e, cudaStreamSynchronize(s));
    return CHD_OK;
}
}  // extern "C"
