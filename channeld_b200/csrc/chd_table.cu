// chd_table.cu — entity-table mode: spawn, move and despawn entities by id (chd_table.cuh).  The host side owns everything that
// must be answered synchronously or assigned deterministically (statuses, id -> slot, free FIFO, quarantine); moves, the
// high-volume path, resolve their ids on the device.
#include "chd_engine.h"

#include "chd_gpu_facing.h"
#include "chd_table.cuh"

#include <unordered_set>

namespace {

// The positions changed: nothing is assigned or built for them yet, and a halo imported before may sit where the high-water mark
// now reaches.  Unlike chd_entities_replaced this keeps handover detection on when the high-water mark grows: the new slots are
// flagged and left out of the handover list.
void touched(chd_engine* e) {
    e->n_own = e->tbl.hw;
    e->n_halo = 0;
    e->halo_on_device = false;
    e->assigned = false;
    e->entities_dirty = true;
}

unsigned grid_for(const chd_engine* e, uint64_t n) {
    return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(blocks_for(n, TBL_THREADS), (uint64_t)e->sm_count * 8));
}

// A pinned staging buffer of at least `bytes` whose last upload has completed (two alternate: a host that spawns every tick waits
// for the copy it made a call earlier, not for the one just enqueued).  The caller records ev_stage[*k] after its copies.
chd_status take_stage(chd_engine* e, uint64_t bytes, int* k, uint8_t** out) {
    chd_engine::Table& t = e->tbl;
    *k = t.next_stage;
    t.next_stage ^= 1;
    CU(e, cudaEventSynchronize(t.ev_stage[*k]));
    if (t.h_stage_cap[*k] < bytes) {
        if (t.h_stage[*k]) CU(e, cudaFreeHost(t.h_stage[*k]));
        t.h_stage[*k] = nullptr;
        t.h_stage_cap[*k] = 0;
        const uint64_t cap = std::max<uint64_t>(bytes, 4096);
        CU(e, cudaHostAlloc((void**)&t.h_stage[*k], cap, cudaHostAllocDefault));
        t.h_stage_cap[*k] = cap;
    }
    *out = t.h_stage[*k];
    return CHD_OK;
}

// An event array on the host: host arrays are read where they are, device arrays are copied back (statuses are synchronous).
template <typename T>
chd_status host_view(chd_engine* e, const T* p, uint32_t n, std::vector<T>& keep, const T** out) {
    *out = p;
    if (!n || !chd_is_device_ptr(e, p)) return CHD_OK;
    keep.resize(n);
    CU(e, cudaMemcpy(keep.data(), p, sizeof(T) * n, cudaMemcpyDeviceToHost));
    *out = keep.data();
    return CHD_OK;
}

chd_status put_status(chd_engine* e, uint8_t* out, const std::vector<uint8_t>& st) {
    if (!out || st.empty()) return CHD_OK;
    if (chd_is_device_ptr(e, out)) {
        CU(e, cudaMemcpy(out, st.data(), st.size(), cudaMemcpyHostToDevice));
    } else {
        memcpy(out, st.data(), st.size());
    }
    return CHD_OK;
}

// The facing storage (include/chd_gpu_facing.h), at the first facing call: every slot has no facing.
chd_status facing_alloc(chd_engine* e) {
    chd_engine::Table& t = e->tbl;
    if (t.d_fx) return CHD_OK;
    const uint64_t N = e->lim.max_entities;
    double *fx = nullptr, *ev = nullptr;
    if (!dalloc(e, &fx, 2 * N) || !dalloc(e, &ev, 2 * N)) return CHD_ERR_CUDA;
    CU(e, cudaMemsetAsync(fx, 0, 16 * N, e->stream));
    t.d_fx = fx;
    t.d_fz = fx + N;
    t.d_ev_face = ev;
    return CHD_OK;
}

// Uploads m (id, slot) pairs and, with positions, their x / z (as doubles) into the device event staging on the engine stream; with
// facings (fx != nullptr) their fx / fz into the facing staging.
chd_status upload_events(chd_engine* e, const std::vector<uint32_t>& id, const std::vector<uint32_t>& slot, const std::vector<double>* x,
                         const std::vector<double>* z, const std::vector<double>* fx = nullptr, const std::vector<double>* fz = nullptr) {
    chd_engine::Table& t = e->tbl;
    const uint64_t m = id.size();
    if (!m) return CHD_OK;
    int k = 0;
    uint8_t* h = nullptr;
    const uint64_t lead = (x ? 16 * m : 0) + (fx ? 16 * m : 0);  // x | z | fx | fz, then id | slot
    chd_status st = take_stage(e, lead + 8 * m, &k, &h);
    if (st != CHD_OK) return st;
    uint32_t* hi = reinterpret_cast<uint32_t*>(h + lead);
    memcpy(hi, id.data(), 4 * m);
    memcpy(hi + m, slot.data(), 4 * m);
    if (x) {
        memcpy(h, x->data(), 8 * m);
        memcpy(h + 8 * m, z->data(), 8 * m);
        CU(e, cudaMemcpyAsync(t.d_ev_pos, h, 16 * m, cudaMemcpyHostToDevice, e->stream));
    }
    if (fx) {
        memcpy(h + 16 * m, fx->data(), 8 * m);
        memcpy(h + 24 * m, fz->data(), 8 * m);
        CU(e, cudaMemcpyAsync(t.d_ev_face, h + 16 * m, 16 * m, cudaMemcpyHostToDevice, e->stream));
    }
    CU(e, cudaMemcpyAsync(t.d_ev, hi, 8 * m, cudaMemcpyHostToDevice, e->stream));
    CU(e, cudaEventRecord(t.ev_stage[k], e->stream));
    return CHD_OK;
}

// The device table from the host map (live entries only: the tombstones go), stream-ordered.
chd_status rebuild_table(chd_engine* e) {
    chd_engine::Table& t = e->tbl;
    std::vector<uint32_t> id, slot;
    id.reserve(t.slot_of.size());
    slot.reserve(t.slot_of.size());
    for (const auto& kv : t.slot_of) {
        id.push_back(kv.first);
        slot.push_back(kv.second);
    }
    CU(e, cudaMemsetAsync(t.d_table, 0, 8ull << t.bits, e->stream));
    chd_status st = upload_events(e, id, slot, nullptr, nullptr);
    if (st != CHD_OK) return st;
    if (!id.empty()) {
        const uint32_t m = (uint32_t)id.size();
        tbl_spawn_kernel<<<grid_for(e, m), TBL_THREADS, 0, e->stream>>>(t.d_table, t.bits, t.d_ev, t.d_ev + m, nullptr, nullptr, m, nullptr, nullptr, nullptr,
                                                                       nullptr);
        KCHECK(e);
    }
    t.used = id.size();
    t.rebuilds++;
    return CHD_OK;
}

bool reserved_id(uint32_t id) { return id == 0u || id == 0xFFFFFFFFu; }

// argument checks of a spawn or a move (at most max_entities moves per call)
chd_status check_events(chd_engine* e, const char* fn, const uint32_t* id, const void* x, const void* z, uint32_t n, bool is_move) {
    if (!e || (n && (!id || !x || !z))) return CHD_ERR_INVALID;
    if (chd_rule_table(e, fn) != CHD_OK) return CHD_ERR_STATE;
    if (is_move && n > e->lim.max_entities) {
        e->fail("%s: %u moves in one call > max_entities %llu", fn, n, (unsigned long long)e->lim.max_entities);
        return CHD_ERR_CAPACITY;
    }
    return CHD_OK;
}

// n values of a host or device array as doubles: the float form widens exactly, as chd_set_entities_f32 does
chd_status widened(chd_engine* e, const void* in, bool f32, uint32_t n, std::vector<double>& out) {
    out.resize(n);
    chd_status st = CHD_OK;
    if (f32) {
        std::vector<float> keep;
        const float* p = nullptr;
        if ((st = host_view(e, (const float*)in, n, keep, &p)) != CHD_OK) return st;
        for (uint32_t i = 0; i < n; i++) out[i] = (double)p[i];
    } else {
        std::vector<double> keep;
        const double* p = nullptr;
        if ((st = host_view(e, (const double*)in, n, keep, &p)) != CHD_OK) return st;
        std::copy(p, p + n, out.begin());
    }
    return CHD_OK;
}

// fx_in == nullptr: no facing (chd_spawn_entities); the facings are written once the storage exists
chd_status spawn(chd_engine* e, const uint32_t* id_in, const void* x_in, const void* z_in, bool f32, uint32_t n, uint8_t* out_status,
                 const void* fx_in = nullptr, const void* fz_in = nullptr) {
    chd_engine::Table& t = e->tbl;
    std::vector<uint32_t> kid;
    const uint32_t* ids = nullptr;
    chd_status st = host_view(e, id_in, n, kid, &ids);
    if (st != CHD_OK) return st;
    std::vector<double> px, pz, pfx, pfz;
    if ((st = widened(e, x_in, f32, n, px)) != CHD_OK || (st = widened(e, z_in, f32, n, pz)) != CHD_OK) return st;
    if (fx_in && ((st = widened(e, fx_in, f32, n, pfx)) != CHD_OK || (st = widened(e, fz_in, f32, n, pfz)) != CHD_OK)) return st;
    std::vector<uint8_t> status(n, (uint8_t)CHD_EV_OK);
    std::vector<uint32_t> aid, aslot;
    std::vector<double> ax, az, afx, afz;
    std::unordered_set<uint32_t> seen;
    seen.reserve(n);
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t id = ids[i];
        uint32_t slot = 0;
        if (reserved_id(id)) {
            status[i] = CHD_EV_RESERVED_ID;
        } else if (!seen.insert(id).second || t.slot_of.count(id)) {
            status[i] = CHD_EV_DUPLICATE;
        } else if (!t.free_fifo.empty()) {
            slot = t.free_fifo.front();
            t.free_fifo.pop_front();
        } else if (t.hw < e->lim.max_entities) {
            slot = t.hw++;
        } else {
            status[i] = CHD_EV_TABLE_FULL;
        }
        if (status[i] != CHD_EV_OK) continue;
        aid.push_back(id);
        aslot.push_back(slot);
        ax.push_back(px[i]);
        az.push_back(pz[i]);
        if (fx_in) {
            afx.push_back(pfx[i]);
            afz.push_back(pfz[i]);
        }
    }
    const uint64_t m = aid.size();
    if (m) {
        StageTimer timer(e, e->stream, CHD_STAGE_ENTITY_EVENTS);
        if ((t.used + m) * 4 > (3ull << t.bits)) {  // live + tombstones would pass 3/4 of the table
            st = rebuild_table(e);
            if (st != CHD_OK) return st;
        }
        for (uint64_t j = 0; j < m; j++) t.slot_of[aid[j]] = aslot[j];
        t.used += m;
        st = upload_events(e, aid, aslot, &ax, &az, fx_in ? &afx : nullptr, fx_in ? &afz : nullptr);
        if (st != CHD_OK) return st;
        tbl_spawn_kernel<<<grid_for(e, m), TBL_THREADS, 0, e->stream>>>(t.d_table, t.bits, t.d_ev, t.d_ev + m, t.d_ev_pos, t.d_ev_pos + m, (uint32_t)m,
                                                                       t.d_id_of_slot, chd_pos_front(e).x, chd_pos_front(e).z, t.d_flag,
                                                                       fx_in ? t.d_ev_face : nullptr, fx_in ? t.d_ev_face + m : nullptr, t.d_fx, t.d_fz);
        KCHECK(e);
        touched(e);
    }
    return put_status(e, out_status, status);
}

// fx == nullptr: the facings stay (chd_move_entities)
chd_status move(chd_engine* e, const uint32_t* id, const void* x, const void* z, bool f32, uint32_t n, const void* fx = nullptr, const void* fz = nullptr) {
    const uint64_t N = e->lim.max_entities;
    chd_engine::Table& t = e->tbl;
    const PosSet& front = chd_pos_front(e);
    cudaStream_t s = e->stream;
    StageTimer timer(e, s, CHD_STAGE_ENTITY_EVENTS);
    // host inputs are copied into the event staging, device inputs read in place
    const uint32_t* did = id;
    if (!chd_is_device_ptr(e, id)) {
        CU(e, cudaMemcpyAsync(t.d_ev, id, 4ull * n, cudaMemcpyDefault, s));
        did = t.d_ev;
    }
    const size_t w = f32 ? sizeof(float) : sizeof(double);
    const void *dx = x, *dz = z;
    if (!(chd_is_device_ptr(e, x) && chd_is_device_ptr(e, z))) {
        uint8_t* base = reinterpret_cast<uint8_t*>(t.d_ev_pos);
        CU(e, cudaMemcpyAsync(base, x, w * n, cudaMemcpyDefault, s));
        CU(e, cudaMemcpyAsync(base + w * N, z, w * n, cudaMemcpyDefault, s));
        dx = base;
        dz = base + w * N;
    }
    const void *dfx = fx, *dfz = fz;
    if (fx && !(chd_is_device_ptr(e, fx) && chd_is_device_ptr(e, fz))) {
        uint8_t* base = reinterpret_cast<uint8_t*>(t.d_ev_face);
        CU(e, cudaMemcpyAsync(base, fx, w * n, cudaMemcpyDefault, s));
        CU(e, cudaMemcpyAsync(base + w * N, fz, w * n, cudaMemcpyDefault, s));
        dfx = base;
        dfz = base + w * N;
    }
    const unsigned grid = grid_for(e, n);
    tbl_move_resolve_kernel<<<grid, TBL_THREADS, 0, s>>>(t.d_table, t.bits, did, n, t.d_mslot, t.d_winner, t.d_stats);
    KCHECK(e);
    if (f32 && fx)
        tbl_move_apply_kernel<float, true><<<grid, TBL_THREADS, 0, s>>>(t.d_mslot, t.d_winner, (const float*)dx, (const float*)dz, n, front.x, front.z, t.d_stats,
                                                                        (const float*)dfx, (const float*)dfz, t.d_fx, t.d_fz);
    else if (fx)
        tbl_move_apply_kernel<double, true><<<grid, TBL_THREADS, 0, s>>>(t.d_mslot, t.d_winner, (const double*)dx, (const double*)dz, n, front.x, front.z,
                                                                         t.d_stats, (const double*)dfx, (const double*)dfz, t.d_fx, t.d_fz);
    else if (f32)
        tbl_move_apply_kernel<float><<<grid, TBL_THREADS, 0, s>>>(t.d_mslot, t.d_winner, (const float*)dx, (const float*)dz, n, front.x, front.z, t.d_stats);
    else
        tbl_move_apply_kernel<double><<<grid, TBL_THREADS, 0, s>>>(t.d_mslot, t.d_winner, (const double*)dx, (const double*)dz, n, front.x, front.z, t.d_stats);
    KCHECK(e);
    touched(e);
    return CHD_OK;
}

chd_status handoff_check(chd_engine* e, const char* fn);
chd_status handoff(chd_engine* e, const char* fn, uint32_t* id, uint32_t* dst_rank, double* x, double* z, double* fx, double* fz, uint32_t cap,
                   uint32_t* count);

template <typename... A>
chd_status refuse(const chd_engine* e, const char* fmt, A... a) {
    e->fail(fmt, a...);
    return CHD_ERR_STATE;
}

}  // namespace

extern "C" {

// ---- The mode rules (DESIGN.md §5, same numbers): entities are named by index, by global id (chd_set_entity_ids) or by table id
// (entity-table mode), visible deltas by index or by global id (id mode).  With them the call-order rules: one query batch per
// interest update (9) and nothing rewritten under a begun chd_begin_interest (13).  Entry points call their rule after the
// argument checks.

// 1. Refused in entity-table mode: the calls that bypass the table (positions, counts, global ids, a slab).
chd_status chd_rule_not_table(chd_engine* e, const char* fn) {
    if (!e->tbl.on) return CHD_OK;
    return refuse(e, "%s is not available in entity-table mode (chd_entity_table_init): use chd_spawn_entities / chd_move_entities / chd_despawn_entities", fn);
}

// 2. The multi-GPU calls take entity-table mode only on an engine made a slab before chd_entity_table_init.
chd_status chd_rule_table_on_slab(chd_engine* e, const char* fn) {
    if (!e->tbl.on || e->slab) return CHD_OK;
    return refuse(e, "%s in entity-table mode needs an engine made a slab (chd_set_slab / chd_comm_init) before chd_entity_table_init", fn);
}

// 3. The calls by id need entity-table mode.
chd_status chd_rule_table(chd_engine* e, const char* fn) { return e->tbl.on ? CHD_OK : refuse(e, "%s before chd_entity_table_init", fn); }

// 4. Entity-table mode starts on a fresh engine; a slab may come first (that is how a table engine becomes a rank of a sharded
// world).  delta_blocked without a slab: chd_set_entity_ids was called, perhaps with NULL.
chd_status chd_rule_fresh_engine(chd_engine* e) {
    if (e->tbl.on || e->built || e->assigned || e->n_own || e->pf_pos.staged >= 0 || e->have_gid || (e->delta_blocked && !e->slab) || e->dl.ids)
        return refuse(e, "chd_entity_table_init needs a fresh engine (no entities set, assigned or built, no chd_set_entity_ids / chd_export_border / "
                         "chd_reserve_visible_delta_ids; chd_set_slab / chd_comm_init may come first)");
    return CHD_OK;
}

// 5. Index-mode deltas are single-GPU only (halo indices are not stable): refused after delta_blocked unless id mode is on.
chd_status chd_rule_index_delta(chd_engine* e) {
    if (!e->delta_blocked || e->dl.ids) return CHD_OK;
    return refuse(e, "index-mode visible deltas are single-GPU only: this engine used chd_set_slab / chd_set_entity_ids / chd_comm_init "
                     "(chd_reserve_visible_delta_ids names entities by global id instead)");
}

// 6. Id mode never follows index mode and keeps its id_space.  In entity-table mode it is the delta mode of slab engines: on one
// GPU the index-mode deltas already name ids.
chd_status chd_rule_id_delta(chd_engine* e, uint32_t id_space) {
    if (e->tbl.on && !e->slab) return chd_rule_not_table(e, "chd_reserve_visible_delta_ids on an engine that is not a slab");
    if (e->dl.on && !e->dl.ids)
        return refuse(e, "chd_reserve_visible_delta_ids: this engine's visible deltas are in index mode (chd_reserve_visible_delta came first)");
    if (!e->dl.on || id_space == e->dl.id_space) return CHD_OK;
    e->fail("chd_reserve_visible_delta_ids: id_space %u differs from the %u the mode was set up with", id_space, e->dl.id_space);
    return CHD_ERR_INVALID;
}

// 7 (after 5). A delta runs after a reserve, in id mode with global ids, on a build of the current state (will_build: built first).
chd_status chd_delta_check(chd_engine* e, bool will_build) {
    if (chd_rule_index_delta(e) != CHD_OK) return CHD_ERR_STATE;
    if (!e->dl.on) return refuse(e, "visible delta before chd_reserve_visible_delta");
    if (e->dl.ids && !e->have_gid && !e->tbl.on) return refuse(e, "id-mode visible delta on an engine without global ids (chd_set_entity_ids)");
    if (will_build) return CHD_OK;
    // id mode: the ids scattered by the delta must be those the build sorted
    if (e->dl.ids && e->entities_dirty)
        return refuse(e, "id-mode visible delta needs a chd_build after the last chd_set_entities / chd_set_entity_ids / chd_import_halo");
    // chd_assign_cells rewrote the keys since the last build: keys and cell CSR no longer describe one state
    if (!e->built || (e->assigned && e->entities_dirty)) return refuse(e, "visible delta needs a chd_build of the current cell assignment");
    // entity-table mode: the ids the lists are translated with must be those of the build the delta measures
    if (e->tbl.on && e->entities_dirty) return refuse(e, "visible delta needs a chd_build after the last spawn / move / despawn");
    return CHD_OK;
}

// 8. The halo import appends to a cell assignment, and its records name entities by global id.
chd_status chd_rule_halo_import(chd_engine* e) {
    if (!e->assigned) return refuse(e, "chd_import_halo before chd_export_border / chd_assign_cells");
    return e->have_gid || e->tbl.on ? CHD_OK : refuse(e, "chd_import_halo requires global entity ids (chd_set_entity_ids or entity-table mode)");
}

// 9. Followers (chd_follow_*) on a slab need entity-table mode: there a follower lives on the rank that owns its entity, which
// the id resolves to through the rank's own table (halo ids never enter it), so the exact position is local.  Index-mode and
// id-mode slabs refuse them (an entity's index there is its place in the host's array plus the halo import order), and an engine
// with followers cannot become a slab (the slab comes first, then chd_entity_table_init, rule 4).  `entity` of a binding is the
// table id in entity-table mode and the entity index otherwise (chd_set_entity_ids does not change that).
chd_status chd_rule_follow(chd_engine* e, const char* fn) {
    if (!e->slab || e->tbl.on) return CHD_OK;
    return refuse(e, "%s: followers on an engine made a slab (chd_set_slab / chd_comm_init) need entity-table mode (chd_entity_table_init after the slab)", fn);
}
chd_status chd_rule_no_followers(chd_engine* e, const char* fn) {
    return e->fw.n_bound ? refuse(e, "%s: %u subscriber slots follow entities (chd_follow_bind); the slab comes before the followers", fn, e->fw.n_bound)
                         : CHD_OK;
}

// ... and one query batch per interest update: a generated batch (chd_follow_queries) and an adopted prefetched one
// (chd_prefetch_queries + chd_adopt_prefetched) exclude each other until the update that consumes the first has been enqueued.
// A generated batch also holds off the reports of the followers it was generated from (chd_get_follow, chd_get_follow_frame).
chd_status chd_rule_no_generated_batch(chd_engine* e, const char* fn) {
    if (!e->fw.ready) return CHD_OK;
    return refuse(e, "%s: the batch generated by chd_follow_queries has not been consumed by an interest update yet (one batch per update)", fn);
}
chd_status chd_rule_one_batch(chd_engine* e, const char* fn) {
    if (chd_rule_no_generated_batch(e, fn) != CHD_OK) return CHD_ERR_STATE;
    if (e->pf_q.cur >= 0) return refuse(e, "%s: the adopted prefetched query batch has not been consumed by an interest update yet", fn);
    return chd_rule_no_chain(e, fn, false);
}

// ... except that chd_follow_queries_with merges the two into one batch: the host part is q or (adopted) the adopted prefetched batch,
// which it consumes.  So an adopted batch is required with q == NULL and refused beside a q.
chd_status chd_rule_merged_batch(chd_engine* e, bool adopted) {
    const char* fn = "chd_follow_queries_with";
    if (chd_rule_no_generated_batch(e, fn) != CHD_OK || chd_rule_no_chain(e, fn, false) != CHD_OK) return CHD_ERR_STATE;
    if (adopted && e->pf_q.cur < 0) return refuse(e, "%s: q == NULL needs chd_prefetch_queries + chd_adopt_prefetched first", fn);
    if (!adopted && e->pf_q.cur >= 0)
        return refuse(e, "%s: the adopted prefetched query batch has not been consumed (pass q == NULL to merge it)", fn);
    return CHD_OK;
}

// ... and an interest update that takes the waiting batch (q == NULL) needs one: with `generated` (CHD_TICK_FOLLOW) the generated
// batch, otherwise either kind.
chd_status chd_rule_batch_waiting(chd_engine* e, const char* fn, bool generated) {
    if (generated) return e->fw.ready ? CHD_OK : refuse(e, "%s: CHD_TICK_FOLLOW without a batch generated by chd_follow_queries", fn);
    if (e->fw.ready || e->pf_q.cur >= 0) return CHD_OK;
    return refuse(e, "%s: q == NULL needs chd_prefetch_queries + chd_adopt_prefetched, or chd_follow_queries, first", fn);
}

// 10. Explicit subscriptions: chd_apply_subscriptions is the whole-world call and chd_apply_subscriptions_sharded the slab call
// (its ops must name cells the slab serves, and reach each rank before the ring limits are exchanged).  Rule 13 as well; the slab
// call follows rule 12's staged updates too (chd_rule_rings_staged, at its call site).
chd_status chd_rule_explicit_subs(chd_engine* e, const char* fn) {
    if (e->slab) return refuse(e, "%s: explicit subscriptions on an engine made a slab (chd_set_slab / chd_comm_init) use chd_apply_subscriptions_sharded", fn);
    return chd_rule_no_chain(e, fn, false);
}
chd_status chd_rule_explicit_subs_slab(chd_engine* e, const char* fn) {
    if (!e->slab) return refuse(e, "%s needs an engine made a slab (chd_set_slab / chd_comm_init); one engine uses chd_apply_subscriptions", fn);
    return chd_rule_no_chain(e, fn, false);
}

// 11. Facings and frames (include/chd_gpu_facing.h) need entity-table mode: index mode's positions come from host snapshots and the
// prefetch pair, and a facing there would be a third pipelined input.  The frame calls follow rule 9 as well.
chd_status chd_rule_facing(chd_engine* e, const char* fn) {
    return e->tbl.on ? CHD_OK : refuse(e, "%s: facings and follower frames need entity-table mode (chd_entity_table_init)", fn);
}

// 12. Ring limits (include/chd_gpu_rings.h) need device-owned rings on a slab, and rule 13 (the chain raises the limits).  A
// communicator engine stages its one chd_rings_append per tick for chd_tick_sharded, which appends after the ring-limit import;
// until then the calls that would append, read or raise around the staged updates are refused.
chd_status chd_rule_ring_limits(chd_engine* e, const char* fn) {
    if (!e->rings.owned || !e->slab) return refuse(e, "%s needs device-owned rings (chd_rings_init) on a slab (chd_set_slab / chd_comm_init)", fn);
    return chd_rule_no_chain(e, fn, false);
}
chd_status chd_rule_rings_staged(chd_engine* e, const char* fn) {
    if (!e->rings.staged) return CHD_OK;
    return refuse(e, "%s: ring updates are staged for the next chd_tick_sharded (one chd_rings_append per tick on a communicator engine)", fn);
}

// 13. chd_begin_interest forks the interest update (and, with_fanout, the fan-out) onto aux_stream, and nothing on the engine
// stream is ordered against that chain until the chd_tick that joins it.  Until then the calls that rewrite what the chain reads,
// or read what it writes, are refused: the interest update reads the query batches, the subscriptions and the channel start times
// and raises the per-cell maxFanOutIntervalMs that chd_rings_append and the ring limits read; the fan-out reads the rings and the
// start times; the follower reports and the adjacent broadcast read the pairs the update rewrites.  `fanout_only`: the call's
// input is read by the fan-out alone (chd_set_rings), so a chain without the fan-out does not exclude it.
chd_status chd_rule_no_chain(chd_engine* e, const char* fn, bool fanout_only) {
    if (!e->interest_pending || (fanout_only && !e->pending_fanout)) return CHD_OK;
    return refuse(e, "%s: chd_begin_interest is pending (not joined by chd_tick yet)", fn);
}

// 14. Byte-carrying device rings (include/chd_gpu_ring_bytes.h).  chd_rings_reserve_bytes comes after chd_rings_init and before any
// append since it, staged or applied (rules 12 and 13 as well).  A byte-carrying engine appends through chd_rings_append_bytes only, so that every entry carries
// its bytes, and an engine without the reservation through chd_rings_append only.  chd_assemble_payloads replays the windows of
// the last fan-out pass over the rings (for_each_selected), so on device rings it needs the reservation and rings that pass read:
// no append applied and no chd_rings_init since it (an append staged on a communicator engine is applied by the next
// chd_tick_sharded, before its fan-out).  The entries' bytes are in the rings, so chd_set_payload_bytes then carries none
// (CHD_ERR_INVALID).
chd_status chd_rule_ring_bytes_reserve(chd_engine* e) {
    const char* fn = "chd_rings_reserve_bytes";
    if (!e->rings.owned) return refuse(e, "%s before chd_rings_init", fn);
    if (e->rings.appended) return refuse(e, "%s after an append: the reservation comes between chd_rings_init and the first append", fn);
    return chd_rule_no_chain(e, fn, false);
}
chd_status chd_rule_ring_append(chd_engine* e, bool bytes) {
    if (e->rings.bytes.on == bytes) return CHD_OK;
    return bytes ? refuse(e, "chd_rings_append_bytes needs byte-carrying rings (chd_rings_reserve_bytes)")
                 : refuse(e, "chd_rings_append on byte-carrying rings (chd_rings_reserve_bytes): every entry carries its bytes (chd_rings_append_bytes)");
}
chd_status chd_rule_assemble_rings(chd_engine* e) {
    if (!e->rings.owned) return CHD_OK;
    if (!e->rings.bytes.on)
        return refuse(e, "chd_assemble_payloads needs host-owned rings (chd_set_rings): payload bytes are indexed by ring position "
                         "(or byte-carrying device rings, chd_rings_reserve_bytes)");
    if (e->rings.after_fanout) return refuse(e, "chd_assemble_payloads: the rings changed after the last fan-out pass (an append or chd_rings_init)");
    return CHD_OK;
}
chd_status chd_rule_payload_entries(chd_engine* e, uint32_t n_entries) {
    if (!n_entries || !e->rings.owned || !e->rings.bytes.on) return CHD_OK;
    e->fail("chd_set_payload_bytes: %u entries on byte-carrying rings (chd_rings_reserve_bytes), whose entries carry their bytes: pass 0", n_entries);
    return CHD_ERR_INVALID;
}

chd_status chd_entity_table_init(chd_engine* e) {
    if (!e) return CHD_ERR_INVALID;
    if (chd_rule_fresh_engine(e) != CHD_OK) return CHD_ERR_STATE;
    chd_engine::Table& t = e->tbl;
    CHD_ENTER(e, ENTRY_DEVICE);
    const uint64_t N = e->lim.max_entities;
    uint32_t bits = 4;
    while ((1ull << bits) < 2 * N) bits++;
    const bool ok = dalloc(e, &t.d_table, 1ull << bits) && dalloc(e, &t.d_id_of_slot, N) && dalloc(e, &t.d_snap_id, N) &&
                    // the padding and alignment of sorted_ent (the emit kernels read it), one per copy-input set
                    dalloc(e, &e->copy_set[0].sorted_id, ((N + 3) / 4) * 4 + 8) && dalloc(e, &e->copy_set[1].sorted_id, ((N + 3) / 4) * 4 + 8) &&
                    dalloc(e, &t.d_winner, N) && dalloc(e, &t.d_mslot, N) && dalloc(e, &t.d_ho_tmp, 3 * N) && dalloc(e, &t.d_build_seq, 2) &&
                    dalloc(e, &t.d_flag, N) && dalloc(e, &t.d_stats, 3) && dalloc(e, &t.d_ev, 2 * N) && dalloc(e, &t.d_ev_pos, 2 * N) &&
                    chd_make_event(e, &t.ev_stage[0]) && chd_make_event(e, &t.ev_stage[1]);
    if (!ok) return CHD_ERR_CUDA;
    cudaStream_t s = e->stream;
    CU(e, cudaMemsetAsync(t.d_table, 0, 8ull << bits, s));
    CU(e, cudaMemsetAsync(t.d_id_of_slot, 0, 4 * N, s));
    CU(e, cudaMemsetAsync(t.d_snap_id, 0, 4 * N, s));
    CU(e, cudaMemsetAsync(t.d_winner, 0, 4 * N, s));
    CU(e, cudaMemsetAsync(t.d_flag, 0, N, s));
    CU(e, cudaMemsetAsync(t.d_stats, 0, 24, s));
    CU(e, cudaMemsetAsync(t.d_build_seq, 0, 8, s));
    CU(e, cudaMemsetAsync(&e->d_ctr->delta_build, 0, 4, s));
    tbl_park_kernel<<<grid_for(e, N), TBL_THREADS, 0, s>>>(chd_pos_front(e).x, chd_pos_front(e).z, (uint32_t)N);  // every slot starts outside the world
    KCHECK(e);
    CU(e, cudaStreamSynchronize(s));
    e->in_place = {};
    t.bits = bits;
    t.on = true;
    return CHD_OK;
}

chd_status chd_spawn_entities(chd_engine* e, const uint32_t* id, const double* x, const double* z, uint32_t n, uint8_t* out_status) {
    const chd_status st = check_events(e, "chd_spawn_entities", id, x, z, n, false);
    if (st != CHD_OK) return st;
    CHD_ENTER(e, ENTRY_DEVICE);
    return spawn(e, id, x, z, false, n, out_status);
}
chd_status chd_spawn_entities_f32(chd_engine* e, const uint32_t* id, const float* x, const float* z, uint32_t n, uint8_t* out_status) {
    const chd_status st = check_events(e, "chd_spawn_entities_f32", id, x, z, n, false);
    if (st != CHD_OK) return st;
    CHD_ENTER(e, ENTRY_DEVICE);
    return spawn(e, id, x, z, true, n, out_status);
}

chd_status chd_despawn_entities(chd_engine* e, const uint32_t* id_in, uint32_t n, uint8_t* out_status) {
    if (!e || (n && !id_in)) return CHD_ERR_INVALID;
    if (chd_rule_table(e, "chd_despawn_entities") != CHD_OK) return CHD_ERR_STATE;
    CHD_ENTER(e, ENTRY_DEVICE);
    chd_engine::Table& t = e->tbl;
    const PosSet& front = chd_pos_front(e);
    std::vector<uint32_t> kid;
    const uint32_t* ids = nullptr;
    chd_status st = host_view(e, id_in, n, kid, &ids);
    if (st != CHD_OK) return st;
    std::vector<uint8_t> status(n, (uint8_t)CHD_EV_OK);
    std::vector<uint32_t> aid, aslot;
    std::unordered_set<uint32_t> seen;
    seen.reserve(n);
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t id = ids[i];
        if (reserved_id(id)) {
            status[i] = CHD_EV_RESERVED_ID;
            continue;
        }
        if (!seen.insert(id).second) {
            status[i] = CHD_EV_DUPLICATE;
            continue;
        }
        auto it = t.slot_of.find(id);
        if (it == t.slot_of.end()) {
            status[i] = CHD_EV_UNKNOWN_ID;
            continue;
        }
        const uint32_t slot = it->second;
        t.slot_of.erase(it);
        aid.push_back(id);
        aslot.push_back(slot);
        // With index-mode visible deltas on, the slot waits until a delta that measured a build without it has succeeded: reused
        // earlier, the snapshot would still hold the old instance there and the delta could not tell the two apart.  Id-mode
        // deltas name ids, not slots: no quarantine.
        if (e->dl.on && !e->dl.ids)
            t.quarantine.push_back(chd_engine::Table::Held{slot, t.builds + 1});
        else
            t.free_fifo.push_back(slot);
    }
    const uint32_t m = (uint32_t)aid.size();
    if (m) {
        StageTimer timer(e, e->stream, CHD_STAGE_ENTITY_EVENTS);
        st = upload_events(e, aid, aslot, nullptr, nullptr);
        if (st != CHD_OK) return st;
        tbl_despawn_kernel<<<grid_for(e, m), TBL_THREADS, 0, e->stream>>>(t.d_table, t.bits, t.d_ev, t.d_ev + m, m, t.d_id_of_slot, front.x, front.z, t.d_flag);
        KCHECK(e);
        touched(e);
    }
    return put_status(e, out_status, status);
}

chd_status chd_move_entities(chd_engine* e, const uint32_t* id, const double* x, const double* z, uint32_t n) {
    const chd_status st = check_events(e, "chd_move_entities", id, x, z, n, true);
    if (st != CHD_OK || !n) return st;
    CHD_ENTER(e, ENTRY_DEVICE);
    return move(e, id, x, z, false, n);
}
chd_status chd_move_entities_f32(chd_engine* e, const uint32_t* id, const float* x, const float* z, uint32_t n) {
    const chd_status st = check_events(e, "chd_move_entities_f32", id, x, z, n, true);
    if (st != CHD_OK || !n) return st;
    CHD_ENTER(e, ENTRY_DEVICE);
    return move(e, id, x, z, true, n);
}

chd_status chd_get_entity_stats(chd_engine* e, chd_entity_stats* out) {
    if (!e || !out) return CHD_ERR_INVALID;
    if (chd_rule_table(e, "chd_get_entity_stats") != CHD_OK) return CHD_ERR_STATE;
    CHD_ENTER(e, ENTRY_COPY_WAIT);
    const chd_engine::Table& t = e->tbl;
    uint64_t* h64 = reinterpret_cast<uint64_t*>(e->h_get);
    CU(e, cudaMemcpyAsync(h64, t.d_stats, 24, cudaMemcpyDeviceToHost, e->stream));
    CU(e, cudaStreamSynchronize(e->stream));
    out->live = (uint32_t)t.slot_of.size();
    out->high_water = t.hw;
    out->quarantined = (uint32_t)t.quarantine.size();
    out->free_slots = (uint32_t)t.free_fifo.size() + (e->lim.max_entities - t.hw);
    out->moves_applied = h64[0];
    out->moves_unknown = h64[1];
    out->moves_superseded = h64[2];
    out->rebuilds = t.rebuilds;
    return CHD_OK;
}

chd_status chd_handoff_entities(chd_engine* e, uint32_t* id, uint32_t* dst_rank, double* x, double* z, uint32_t cap, uint32_t* count) {
    if (!e || !count || (cap && (!id || !dst_rank || !x || !z))) return CHD_ERR_INVALID;
    if (handoff_check(e, "chd_handoff_entities") != CHD_OK) return CHD_ERR_STATE;
    CHD_ENTER(e, ENTRY_DEVICE);
    return handoff(e, "chd_handoff_entities", id, dst_rank, x, z, nullptr, nullptr, cap, count);
}

chd_status chd_handoff_entities_facing(chd_engine* e, uint32_t* id, uint32_t* dst_rank, double* x, double* z, double* fx, double* fz, uint32_t cap,
                                       uint32_t* count) {
    if (!e || !count || (cap && (!id || !dst_rank || !x || !z || !fx || !fz))) return CHD_ERR_INVALID;
    if (chd_rule_facing(e, "chd_handoff_entities_facing") != CHD_OK || handoff_check(e, "chd_handoff_entities_facing") != CHD_OK) return CHD_ERR_STATE;
    CHD_ENTER(e, ENTRY_DEVICE);
    const chd_status st = facing_alloc(e);
    if (st != CHD_OK) return st;
    return handoff(e, "chd_handoff_entities_facing", id, dst_rank, x, z, fx, fz, cap, count);
}

// ---- facings (include/chd_gpu_facing.h)

chd_status chd_spawn_entities_facing(chd_engine* e, const uint32_t* id, const double* x, const double* z, const double* fx, const double* fz, uint32_t n,
                                     uint8_t* out_status) {
    if (e && n && (!fx || !fz)) return CHD_ERR_INVALID;
    chd_status st = check_events(e, "chd_spawn_entities_facing", id, x, z, n, false);
    if (st != CHD_OK) return st;
    CHD_ENTER(e, ENTRY_DEVICE);
    if ((st = facing_alloc(e)) != CHD_OK) return st;
    return spawn(e, id, x, z, false, n, out_status, fx, fz);
}
chd_status chd_spawn_entities_facing_f32(chd_engine* e, const uint32_t* id, const float* x, const float* z, const float* fx, const float* fz, uint32_t n,
                                         uint8_t* out_status) {
    if (e && n && (!fx || !fz)) return CHD_ERR_INVALID;
    chd_status st = check_events(e, "chd_spawn_entities_facing_f32", id, x, z, n, false);
    if (st != CHD_OK) return st;
    CHD_ENTER(e, ENTRY_DEVICE);
    if ((st = facing_alloc(e)) != CHD_OK) return st;
    return spawn(e, id, x, z, true, n, out_status, fx, fz);
}

chd_status chd_move_entities_facing(chd_engine* e, const uint32_t* id, const double* x, const double* z, const double* fx, const double* fz, uint32_t n) {
    if (e && n && (!fx || !fz)) return CHD_ERR_INVALID;
    chd_status st = check_events(e, "chd_move_entities_facing", id, x, z, n, true);
    if (st != CHD_OK) return st;
    CHD_ENTER(e, ENTRY_DEVICE);
    if ((st = facing_alloc(e)) != CHD_OK || !n) return st;
    return move(e, id, x, z, false, n, fx, fz);
}
chd_status chd_move_entities_facing_f32(chd_engine* e, const uint32_t* id, const float* x, const float* z, const float* fx, const float* fz, uint32_t n) {
    if (e && n && (!fx || !fz)) return CHD_ERR_INVALID;
    chd_status st = check_events(e, "chd_move_entities_facing_f32", id, x, z, n, true);
    if (st != CHD_OK) return st;
    CHD_ENTER(e, ENTRY_DEVICE);
    if ((st = facing_alloc(e)) != CHD_OK || !n) return st;
    return move(e, id, x, z, true, n, fx, fz);
}

}  // extern "C"

namespace {

// the mode rule and the call order of a hand-off
chd_status handoff_check(chd_engine* e, const char* fn) {
    if (chd_rule_table(e, fn) != CHD_OK) return CHD_ERR_STATE;
    if (!e->assigned) {
        // the keys must describe the current positions: a spawn, move, despawn or hand-off since the last assignment changed them
        e->fail("%s needs a cell assignment after the last spawn / move / despawn / hand-off (chd_export_border, chd_assign_cells, chd_build or a "
                "tick)", fn);
        return CHD_ERR_STATE;
    }
    return CHD_OK;
}

// chd_handoff_entities(_facing), named fn in errors: fx == nullptr lists no facings
chd_status handoff(chd_engine* e, const char* fn, uint32_t* id, uint32_t* dst_rank, double* x, double* z, double* fx, double* fz, uint32_t cap,
                   uint32_t* count) {
    chd_engine::Table& t = e->tbl;
    const PosSet& front = chd_pos_front(e);
    cudaStream_t s = e->stream;
    const uint64_t N = e->lim.max_entities;
    const uint32_t world = e->comm ? (uint32_t)e->comm_world : 1u;
    // the list goes to the event staging (free between calls: every user is on this stream) and the radix sort's temporaries
    uint32_t *d_id = t.d_ev, *d_slot = t.d_ev + N, *d_dst = e->ent_sort.tmp_val;
    double *d_hx = t.d_ev_pos, *d_hz = t.d_ev_pos + N;
    chd_status st = chd_epoch_tick(e, s, EP_BORDER);
    if (st != CHD_OK) return st;
    bump_epoch_kernel<<<1, 1, 0, s>>>(e->d_epoch + EP_BORDER);
    KCHECK(e);
    HandoffSink sink{e->g, world, e->d_key, chd_entity_ids(e), front.x, front.z, d_id, d_slot, d_dst, d_hx, d_hz, e->d_boff};
    if (fx) {  // the facings go to the facing staging, copied out before the despawn pass below removes the entities
        sink.pfx = t.d_fx;
        sink.pfz = t.d_fz;
        sink.fx = t.d_ev_face;
        sink.fz = t.d_ev_face + N;
    }
    SCAN(e, compact_1p(HandoffFlag{e->g, e->d_key}, sink, e->n_own, e->site_border, s));
    st = chd_read_u32(e, e->d_boff, count);
    if (st != CHD_OK) return st;
    const uint32_t m = *count;
    if (m > cap) {  // transactional: nothing removed, a repeat call with a larger buffer lists the same entities
        e->fail("%s: %u entities to hand off > cap %u", fn, m, cap);
        return CHD_ERR_CAPACITY;
    }
    if (!m) return CHD_OK;
    CU(e, cudaMemcpyAsync(id, d_id, 4ull * m, cudaMemcpyDefault, s));
    CU(e, cudaMemcpyAsync(dst_rank, d_dst, 4ull * m, cudaMemcpyDefault, s));
    CU(e, cudaMemcpyAsync(x, d_hx, 8ull * m, cudaMemcpyDefault, s));
    CU(e, cudaMemcpyAsync(z, d_hz, 8ull * m, cudaMemcpyDefault, s));
    if (fx) {
        CU(e, cudaMemcpyAsync(fx, t.d_ev_face, 8ull * m, cudaMemcpyDefault, s));
        CU(e, cudaMemcpyAsync(fz, t.d_ev_face + N, 8ull * m, cudaMemcpyDefault, s));
    }
    std::vector<uint32_t> hid(m), hslot(m);
    CU(e, cudaMemcpyAsync(hid.data(), d_id, 4ull * m, cudaMemcpyDeviceToHost, s));
    CU(e, cudaMemcpyAsync(hslot.data(), d_slot, 4ull * m, cudaMemcpyDeviceToHost, s));
    CU(e, cudaStreamSynchronize(s));
    // The ids live on at their new owner: the slots are free at once (no quarantine), in slot order.  The apply pass is a
    // despawn's (tombstone, slot -> id cleared, slot parked and flagged), so neither rank reports the hand-off as a handover.
    for (uint32_t j = 0; j < m; j++) {
        t.slot_of.erase(hid[j]);
        t.free_fifo.push_back(hslot[j]);
    }
    StageTimer timer(e, s, CHD_STAGE_ENTITY_EVENTS);
    tbl_despawn_kernel<<<grid_for(e, m), TBL_THREADS, 0, s>>>(t.d_table, t.bits, d_id, d_slot, m, t.d_id_of_slot, front.x, front.z, t.d_flag);
    KCHECK(e);
    touched(e);
    return CHD_OK;
}

}  // namespace

extern "C" {

// After every table-mode build into copy-input set `c`, on the build's stream: its id-valued sorted entity array and, after a fresh
// cell assignment, the handover list in ids without the slots spawned or despawned since the previous one (then the flags clear).
chd_status chd_table_after_build(chd_engine* e, cudaStream_t s, const CopySet& c) {
    chd_engine::Table& t = e->tbl;
    if (!t.on) return CHD_OK;
    // on slabs the build's length (own slots + halo records) lives on the device
    const uint32_t* n_ptr = e->halo_on_device ? e->d_n_build : nullptr;
    const uint32_t n = e->halo_on_device ? e->lim.max_entities : e->n_own + e->n_halo;
    const EntityIds ids = chd_entity_ids(e);
    const bool raw = t.ho_raw;
    const uint64_t key = stage_key(0x7461626c65ull, n, n_ptr, ids.own, ids.gid, raw, c.sorted_ent, c.sorted_id, ids.own_ids, e->ho_cap);
    const unsigned grid = (unsigned)e->sm_count * 4;
    chd_status st = run_stage(e, s, t.g_post, key, [&]() -> chd_status {
        tbl_gather_ids_kernel<<<grid, TBL_THREADS, 0, s>>>(c.sorted_ent, ids, n, n_ptr, c.sorted_id, t.d_build_seq);
        KCHECK(e);
        if (!raw) return CHD_OK;
        const HandoverOut ho{e->d_ho_entity, e->d_ho_src, e->d_ho_dst, &e->d_ctr->n_handover, e->ho_cap};
        tbl_handover_stash_kernel<<<grid, TBL_THREADS, 0, s>>>(ho, t.d_ho_tmp, t.d_build_seq + 1);
        KCHECK(e);
        CU(e, cudaMemsetAsync(&e->d_ctr->n_handover, 0, 4, s));
        tbl_handover_ids_kernel<<<grid, TBL_THREADS, 0, s>>>(ho, t.d_ho_tmp, t.d_build_seq + 1, t.d_flag, ids);
        KCHECK(e);
        if (e->n_own) CU(e, cudaMemsetAsync(t.d_flag, 0, e->n_own, s));
        return CHD_OK;
    });
    if (st != CHD_OK) return st;
    t.builds++;
    t.ho_raw = false;
    return CHD_OK;
}

// Inside the visible-delta stage, after the write pass: enter / leave lists from slots to ids, then the snapshot's ids advance.
chd_status chd_table_delta_ids(chd_engine* e, cudaStream_t s) {
    chd_engine::Table& t = e->tbl;
    const chd_engine::Delta& D = e->dl;
    const unsigned grid = (unsigned)e->sm_count * 8;
    const EntityIds ids = chd_entity_ids(e);  // (index mode runs on one GPU: every position is a slot below the high-water mark)
    tbl_delta_ids_kernel<<<grid, TBL_THREADS, 0, s>>>(D.enter_off, D.leave_off, D.n_out, D.enter_cap, D.leave_cap, D.enter, D.leave, ids, t.d_snap_id,
                                                      t.d_build_seq, &e->d_ctr->delta_build);
    KCHECK(e);
    tbl_delta_commit_kernel<<<grid, TBL_THREADS, 0, s>>>(D.enter_off, D.leave_off, D.n_out, D.enter_cap, D.leave_cap, ids, e->n_sorted, t.d_snap_id);
    KCHECK(e);
    return CHD_OK;
}

// A summary the host decoded says that the last successful delta measured build `delta_build`: the slots despawned before that
// build are out of every snapshot a later delta compares against, so they may be reused.
void chd_table_observe(chd_engine* e, uint32_t delta_build) {
    chd_engine::Table& t = e->tbl;
    while (!t.quarantine.empty() && t.quarantine.front().build <= delta_build) {
        t.free_fifo.push_back(t.quarantine.front().slot);
        t.quarantine.pop_front();
    }
}
}  // extern "C"
