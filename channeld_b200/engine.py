"""Thin object wrapper over the C ABI (include/chd_gpu.h).  No compute happens in Python: every method is one
C call; results come back as numpy arrays copied by the library.  Inputs may be numpy arrays (host), torch
tensors (pinned host or CUDA) or raw addresses.
"""
import ctypes as C

import numpy as np

from . import capi
from .capi import ChdError, GridCfg, Limits, QueryBatch, TickSummary, ptr

SPATIAL_CHANNEL_ID_START = 0x10000  # settings.go:94
ENTITY_CHANNEL_ID_START = 0x80000   # settings.go:95


def grid_cfg(offx, offz, w, h, cols, rows, server_cols=1, server_rows=1, border=0, id_start=SPATIAL_CHANNEL_ID_START):
    return GridCfg(float(offx), float(offz), float(w), float(h), int(cols), int(rows), int(server_cols), int(server_rows),
                   int(border), int(id_start))


def make_batch(n, sub=None, kind=None, sphere=None, box=None, cone=None, spots=None, keep=None):
    """Builds a chd_query_batch.  sphere=(cx,cz,r) box=(cx,cz,ex,ez) cone=(cx,cz,dx,dz,angle,r) are tuples of
    arrays; spots=(spot_off, spot_ndist, x, z, dist).  Arrays are kept alive in `keep` (a list)."""
    keep = keep if keep is not None else []
    b = QueryBatch()
    b.n = int(n)

    def f64(a):
        if a is None:
            return None
        if isinstance(a, np.ndarray):
            a = np.ascontiguousarray(a, np.float64)
        keep.append(a)
        return ptr(a)

    def u32(a):
        if a is None:
            return None
        if isinstance(a, np.ndarray):
            a = np.ascontiguousarray(a, np.uint32)
        keep.append(a)
        return ptr(a)

    b.sub = u32(sub)
    if kind is not None:
        if isinstance(kind, np.ndarray):
            kind = np.ascontiguousarray(kind, np.uint8)
        keep.append(kind)
        b.kind = ptr(kind)
    if sphere is not None:
        b.sph_cx, b.sph_cz, b.sph_r = (f64(a) for a in sphere)
    if box is not None:
        b.box_cx, b.box_cz, b.box_ex, b.box_ez = (f64(a) for a in box)
    if cone is not None:
        b.cone_cx, b.cone_cz, b.cone_dx, b.cone_dz, b.cone_angle, b.cone_r = (f64(a) for a in cone)
    if spots is not None:
        off, ndist, x, z, dist = spots
        b.spot_off, b.spot_ndist, b.spot_x, b.spot_z, b.spot_dist = u32(off), u32(ndist), f64(x), f64(z), u32(dist)
    return b, keep


def host_part_size(n_h):
    """H of chd_follow_queries_with: the size class of a host part of n_h entries (0, or max(256, the next power of two >= n_h)).
    The followers' entries of the merged batch, and of its status list, start at H."""
    n_h = int(n_h)
    return 0 if n_h == 0 else max(256, 1 << (n_h - 1).bit_length())


class Engine:
    def __init__(self, cfg, n_entities, n_subscribers, device=0, **limit_overrides):
        self.L = capi.lib()
        self.cfg = cfg
        lim = Limits()
        self.L.chd_default_limits(C.byref(cfg), int(n_entities), int(n_subscribers), C.byref(lim))
        for k, v in limit_overrides.items():
            if not hasattr(lim, k):
                raise KeyError(k)
            setattr(lim, k, v)
        self.lim = lim
        h = C.c_void_p()
        st = self.L.chd_create(C.byref(cfg), C.byref(lim), int(device), C.byref(h))
        if st != capi.OK:
            raise ChdError(st, self.L.chd_last_error(None).decode())
        self.h = h
        self.n_cells = cfg.grid_cols * cfg.grid_rows
        self.n_slots = 0
        self._keep = []

    def close(self):
        if getattr(self, "h", None):
            self.L.chd_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, st):
        if st != capi.OK:
            raise ChdError(st, self.L.chd_last_error(self.h).decode())

    # ---- plumbing
    def set_stream(self, cuda_stream):
        self._ck(self.L.chd_set_stream(self.h, cuda_stream))

    def sync(self):
        self._ck(self.L.chd_sync(self.h))

    # ---- GetChannelId (batched)
    def cell_of(self, x, z, with_valid=False):
        x = np.ascontiguousarray(x, np.float64)
        z = np.ascontiguousarray(z, np.float64)
        out = np.zeros(len(x), np.uint32)
        if with_valid:
            ok = np.zeros(len(x), np.uint8)
            self._ck(self.L.chd_cell_of_valid(self.h, ptr(x), ptr(z), len(x), ptr(out), ptr(ok)))
            return out, ok.astype(bool)
        self._ck(self.L.chd_cell_of(self.h, ptr(x), ptr(z), len(x), ptr(out)))
        return out

    # ---- entities / build
    def _upload_positions(self, fn, keep, dtype, x, z, n):
        # numpy arrays are converted to `dtype`; the H2D copy is asynchronous, so the arrays stay referenced in `keep` until
        # the next upload of the same kind
        if isinstance(x, np.ndarray):
            x = np.ascontiguousarray(x, dtype)
            z = np.ascontiguousarray(z, dtype)
        n = len(x) if n is None else n
        setattr(self, keep, [x, z])
        self._ck(fn(self.h, ptr(x), ptr(z), int(n)))

    def set_entities(self, x, z, n=None):
        self._upload_positions(self.L.chd_set_entities, "_keep", np.float64, x, z, n)

    def prefetch_entities(self, x, z, n=None):
        """Start the H2D upload of the NEXT tick's positions (overlaps the tick in flight); see chd_prefetch_entities."""
        self._upload_positions(self.L.chd_prefetch_entities, "_keep_prefetch", np.float64, x, z, n)

    def set_entities_f32(self, x, z, n=None):
        """Positions that are floats at the source (unrealpb.FVector): uploaded as floats, widened exactly on the device."""
        self._upload_positions(self.L.chd_set_entities_f32, "_keep", np.float32, x, z, n)

    def prefetch_entities_f32(self, x, z, n=None):
        self._upload_positions(self.L.chd_prefetch_entities_f32, "_keep_prefetch", np.float32, x, z, n)

    def adopt_prefetched(self):
        self._ck(self.L.chd_adopt_prefetched(self.h))
        self._keep = getattr(self, "_keep_prefetch", None)

    def set_entity_ids(self, gid):
        if gid is None:
            self._ck(self.L.chd_set_entity_ids(self.h, None, 0))
            return
        if isinstance(gid, np.ndarray):
            gid = np.ascontiguousarray(gid, np.uint32)
        self._keep_gid = gid
        self._ck(self.L.chd_set_entity_ids(self.h, ptr(gid), len(gid)))

    def entity_buffers(self):
        dx, dz, n = C.c_void_p(), C.c_void_p(), C.c_uint32()
        self._ck(self.L.chd_entity_buffers(self.h, C.byref(dx), C.byref(dz), C.byref(n)))
        return dx.value, dz.value, n.value

    def set_entity_count(self, n):
        self._ck(self.L.chd_set_entity_count(self.h, int(n)))

    def assign_cells(self):
        self._ck(self.L.chd_assign_cells(self.h))

    def build(self):
        self._ck(self.L.chd_build(self.h))

    # ---- subscribers / interest
    def set_subscribers(self, conn_id):
        conn_id = np.ascontiguousarray(conn_id, np.uint32)
        self._keep_conn = conn_id
        self._ck(self.L.chd_set_subscribers(self.h, ptr(conn_id), len(conn_id)))
        self.n_slots = len(conn_id)

    def add_subscribers(self, slots, conn_ids):
        slots = np.ascontiguousarray(slots, np.uint32)
        conn_ids = np.ascontiguousarray(conn_ids, np.uint32)
        self._ck(self.L.chd_add_subscribers(self.h, ptr(slots), ptr(conn_ids), len(slots)))
        if len(slots):
            self.n_slots = max(self.n_slots, int(slots.max()) + 1)

    def remove_subscribers(self, slots):
        slots = np.ascontiguousarray(slots, np.uint32)
        self._ck(self.L.chd_remove_subscribers(self.h, ptr(slots), len(slots)))

    def apply_subscriptions(self, slots, channel_ids, ops, interval=None, delay=None, skip_self=None, skip_first=None, now_ns=0, present=None,
                            status=True):
        """SUB_TO_CHANNEL / UNSUB_FROM_CHANNEL for spatial channels (include/chd_gpu_subs.h), applied in array order at now_ns.
        Each option is None (no op carries it) or one value per op; `present` (CHD_SUBOPT_* per op) says which ops carry which
        option, and defaults to every given option on every op.  Returns the CHD_SUB_* status per op (None with status=False, which
        adds no host synchronisation)."""
        return self._subs(self.L.chd_apply_subscriptions, slots, channel_ids, ops, interval, delay, skip_self, skip_first, now_ns, present,
                          status)

    def apply_subscriptions_sharded(self, slots, channel_ids, ops, interval=None, delay=None, skip_self=None, skip_first=None, now_ns=0,
                                    present=None, status=True):
        """apply_subscriptions on a slab engine (include/chd_gpu_subs_sharded.h): a SUB of a cell outside the served columns gets
        SUB_ERR_OUTSIDE_SLAB.  sharding.route_sub_ops splits a batch named by subscriber keys into the ranks' batches."""
        return self._subs(self.L.chd_apply_subscriptions_sharded, slots, channel_ids, ops, interval, delay, skip_self, skip_first, now_ns,
                          present, status)

    def _subs(self, fn, slots, channel_ids, ops, interval, delay, skip_self, skip_first, now_ns, present, status):
        slots = np.ascontiguousarray(slots, np.uint32)
        n = len(slots)
        arrs = dict(slot=slots, channel_id=np.ascontiguousarray(channel_ids, np.uint32), op=np.ascontiguousarray(ops, np.uint8))
        mask = np.zeros(n, np.uint8)
        for name, v, dt, bit in (("interval_ms", interval, np.uint32, capi.SUBOPT_INTERVAL), ("delay_ms", delay, np.int32, capi.SUBOPT_DELAY),
                                 ("skip_self", skip_self, np.uint8, capi.SUBOPT_SKIP_SELF), ("skip_first", skip_first, np.uint8, capi.SUBOPT_SKIP_FIRST)):
            if v is not None:
                arrs[name] = np.ascontiguousarray(np.broadcast_to(np.asarray(v).astype(dt), (n,)))
                mask |= bit
        arrs["present"] = mask if present is None else np.ascontiguousarray(present, np.uint8)
        assert all(len(a) == n for a in arrs.values())
        b = capi.SubBatch(n=n, **{k: ptr(a) for k, a in arrs.items()})
        self._keep_subs = arrs  # (the copies are asynchronous without out_status)
        out = np.zeros(n, np.uint8) if status else None
        self._ck(fn(self.h, C.byref(b), int(now_ns), ptr(out)))
        return out

    def query_channel_ids(self, batch, cap=None):
        """-> (status[n], off[n+1], channel_id[], dist[])"""
        n = batch.n
        cap = int(cap if cap is not None else self.lim.max_pairs)
        status = np.zeros(n, np.uint32)
        off = np.zeros(n + 1, np.uint32)
        ids = np.zeros(cap, np.uint32)
        dist = np.zeros(cap, np.uint32)
        self._ck(self.L.chd_query_channel_ids(self.h, C.byref(batch), ptr(status), ptr(off), ptr(ids), ptr(dist), cap))
        t = int(off[n]) if n else 0
        return status, off, ids[:t].copy(), dist[:t].copy()

    def update_interest(self, batch, now_ns):
        self._ck(self.L.chd_update_interest(self.h, C.byref(batch) if batch is not None else None, int(now_ns)))

    def emit_visible(self):
        self._ck(self.L.chd_emit_visible(self.h))

    def _upload_rings(self, fn, keep, ring_off, arrival, sender, index, channel_msg_index):
        # the arrays stay referenced in `keep` until the next upload of the same kind (asynchronous H2D)
        ring_off = np.ascontiguousarray(ring_off, np.uint32)
        arrival = np.ascontiguousarray(arrival, np.int64)
        sender = np.ascontiguousarray(sender, np.uint32)
        index = np.ascontiguousarray(index, np.uint64)
        cmi = None if channel_msg_index is None else np.ascontiguousarray(channel_msg_index, np.uint64)
        setattr(self, keep, [ring_off, arrival, sender, index, cmi])
        self._ck(fn(self.h, ptr(ring_off), int(ring_off[-1]), ptr(arrival), ptr(sender), ptr(index), ptr(cmi)))

    def set_rings(self, ring_off, arrival, sender, index, channel_msg_index=None):
        self._upload_rings(self.L.chd_set_rings, "_keep_ring", ring_off, arrival, sender, index, channel_msg_index)

    # ---- device-owned rings (ChannelData.OnUpdate's buffer maintenance on the device)
    def rings_init(self, capacity_per_cell):
        self._ck(self.L.chd_rings_init(self.h, int(capacity_per_cell)))

    def rings_append(self, upd_off, arrival, sender, n=None):
        """Appends updates given as a CSR by cell (upd_off: C + 1 offsets).  n: the update count, upd_off[-1] by default; the
        device reads no update at or past n, whatever upd_off says."""
        upd_off = np.ascontiguousarray(upd_off, np.uint32)
        arrival = np.ascontiguousarray(arrival, np.int64)
        sender = np.ascontiguousarray(sender, np.uint32)
        n = int(upd_off[-1]) if n is None else int(n)
        self._ck(self.L.chd_rings_append(self.h, ptr(upd_off), n, ptr(arrival) if n else None, ptr(sender) if n else None))

    def _ring_off(self):
        """the live entries' CSR by cell (C + 1 offsets)"""
        off = np.zeros(self.n_cells + 1, np.uint32)
        self._ck(self.L.chd_get_rings(self.h, ptr(off), None, None, None, None, 0))
        return off

    def get_rings(self):
        """-> dict(off, arrival, sender, index, msg_index): every live entry in ring order, CSR by cell, and each channel's msgIndex"""
        off = self._ring_off()
        n = int(off[-1])
        arr, snd, idx = np.zeros(n + 1, np.int64), np.zeros(n + 1, np.uint32), np.zeros(n + 1, np.uint64)
        cmi = np.zeros(self.n_cells, np.uint64)
        self._ck(self.L.chd_get_rings(self.h, ptr(off), ptr(arr), ptr(snd), ptr(idx), ptr(cmi), n))
        return dict(off=off, arrival=arr[:n], sender=snd[:n], index=idx[:n], msg_index=cmi)

    def fanout_tick(self, t_ns):
        self._ck(self.L.chd_fanout_tick(self.h, int(t_ns)))

    def summary(self):
        s = TickSummary()
        self._ck(self.L.chd_summary(self.h, C.byref(s)))
        return s

    def begin_interest(self, batch, t_ns, with_fanout=True):
        """batch None = the batch handed over by prefetch_queries + adopt_prefetched."""
        self._ck(self.L.chd_begin_interest(self.h, C.byref(batch) if batch is not None else None, int(t_ns), int(bool(with_fanout))))

    def prefetch_queries(self, batch, keep=None):
        self._keep_pf_q = (batch, keep)
        self._ck(self.L.chd_prefetch_queries(self.h, C.byref(batch)))

    def prefetch_rings(self, ring_off, arrival, sender, index, channel_msg_index=None):
        self._upload_rings(self.L.chd_prefetch_rings, "_keep_pf_ring", ring_off, arrival, sender, index, channel_msg_index)

    def tick(self, batch, t_ns, flags=capi.TICK_ALL, want_summary=True):
        s = TickSummary() if want_summary else None
        self._ck(self.L.chd_tick(self.h, C.byref(batch) if batch is not None else None, int(t_ns), int(flags),
                                 C.byref(s) if s is not None else None))
        return s

    # ---- results
    def get_cells(self):
        cs = np.zeros(self.n_cells + 1, np.uint32)
        self._ck(self.L.chd_get_cells(self.h, ptr(cs), None))
        se = np.zeros(int(cs[-1]), np.uint32)
        self._ck(self.L.chd_get_cells(self.h, None, ptr(se)))
        return cs, se

    def get_pairs(self, n_pairs=None):
        if n_pairs is None:
            off = np.zeros(self.n_slots + 1, np.uint32)
            self._ck(self.L.chd_get_pairs(self.h, ptr(off), None, None, None, None, None, None))
            n_pairs = int(off[-1])
        P = int(n_pairs)
        off = np.zeros(self.n_slots + 1, np.uint32)
        ch = np.zeros(P, np.uint32); dist = np.zeros(P, np.uint32); iv = np.zeros(P, np.uint32)
        fl = np.zeros(P, np.uint8); last = np.zeros(P, np.int64); li = np.zeros(P, np.uint64)
        self._ck(self.L.chd_get_pairs(self.h, ptr(off), ptr(ch), ptr(dist), ptr(iv), ptr(fl), ptr(last), ptr(li)))
        return dict(off=off, channel=ch, dist=dist, interval=iv, flags=fl, last=last, last_index=li)

    def get_query_status(self, n):
        st = np.zeros(n, np.uint32)
        self._ck(self.L.chd_get_query_status(self.h, ptr(st), n))
        return st

    def get_diff(self, n_new, n_unsub):
        a = np.zeros(n_new, np.uint32); b = np.zeros(n_new, np.uint32)
        c = np.zeros(n_unsub, np.uint32); d = np.zeros(n_unsub, np.uint32)
        self._ck(self.L.chd_get_diff(self.h, ptr(a), ptr(b), ptr(c), ptr(d)))
        return (a, b), (c, d)

    def get_visible(self, n_visible=None):
        off = np.zeros(self.n_slots + 1, np.uint64)
        self._ck(self.L.chd_get_visible(self.h, ptr(off), None))
        V = int(off[-1]) if n_visible is None else int(n_visible)
        ve = np.zeros(V, np.uint32)
        self._ck(self.L.chd_get_visible(self.h, None, ptr(ve)))
        return off, ve

    def get_visible_slot(self, slot, cap=1 << 20):
        out = np.zeros(cap, np.uint32)
        n = C.c_uint64()
        self._ck(self.L.chd_get_visible_slot(self.h, int(slot), ptr(out), cap, C.byref(n)))
        if n.value > cap:
            return self.get_visible_slot(slot, int(n.value))
        return out[:n.value].copy()

    def get_due(self, n_due):
        out = np.zeros(int(n_due), capi.DUE_DTYPE)
        if n_due:
            self._ck(self.L.chd_get_due(self.h, ptr(out), int(n_due)))
        return out

    def get_handover(self, n):
        a = np.zeros(n, np.uint32); b = np.zeros(n, np.uint32); c = np.zeros(n, np.uint32)
        self._ck(self.L.chd_get_handover(self.h, ptr(a), ptr(b), ptr(c), n))
        return a, b, c

    def due_classes(self, n_due):
        """Window classes of the last fan-out pass -> (class_of[n_due], class_rep[n_classes], class_count[n_classes])."""
        of = np.zeros(n_due, np.uint32)
        rep = np.zeros(max(n_due, 1), np.uint32)
        cnt = np.zeros(max(n_due, 1), np.uint32)
        n = C.c_uint32(0)
        self._ck(self.L.chd_due_classes(self.h, ptr(of), ptr(rep), ptr(cnt), len(rep), C.byref(n)))
        return of, rep[:n.value], cnt[:n.value]

    def set_subscriber_types(self, conn_type):
        if conn_type is None:
            self._ck(self.L.chd_set_subscriber_types(self.h, None, 0))
            return
        t = np.ascontiguousarray(conn_type, np.uint8)
        self._ck(self.L.chd_set_subscriber_types(self.h, ptr(t), len(t)))

    def adjacent_broadcast(self, channel_id, broadcast, sender_conn_id=None, client_conn_id=None, cap=None):
        """BroadcastType_ADJACENT_CHANNELS recipient sets (message.go:188-239) -> (status[n], off[n+1], slot[])."""
        ch = np.ascontiguousarray(channel_id, np.uint32)
        bc = np.ascontiguousarray(broadcast, np.uint32)
        n = len(ch)
        snd = None if sender_conn_id is None else np.ascontiguousarray(sender_conn_id, np.uint32)
        cli = None if client_conn_id is None else np.ascontiguousarray(client_conn_id, np.uint32)
        b = capi.BroadcastBatch()
        b.n, b.channel_id, b.broadcast, b.sender_conn_id, b.client_conn_id = n, ptr(ch), ptr(bc), ptr(snd), ptr(cli)
        cap = int(cap if cap is not None else max(1, 9 * n * max(self.n_slots, 1)))
        cap = min(cap, 1 << 26)
        status, off, slot = np.zeros(n, np.uint32), np.zeros(n + 1, np.uint32), np.zeros(cap, np.uint32)
        self._ck(self.L.chd_adjacent_broadcast(self.h, C.byref(b), ptr(status), ptr(off), ptr(slot), cap))
        return status, off, slot[:off[-1]]

    # ---- visible-set deltas (entered / left entities per subscriber slot since the last successful delta)
    def reserve_visible_delta(self, cap_entries):
        self._ck(self.L.chd_reserve_visible_delta(self.h, int(cap_entries)))

    def reserve_visible_delta_ids(self, cap_entries, id_space):
        """Id mode: the deltas name global ids in [0, id_space) (chd_set_entity_ids, halo records); works on slabs too."""
        self._ck(self.L.chd_reserve_visible_delta_ids(self.h, int(cap_entries), int(id_space)))

    def visible_delta(self):
        self._ck(self.L.chd_visible_delta(self.h))

    def visible_delta_counts(self):
        """-> (n_entered, n_left, n_slots) of the last delta (the required sizes when it overflowed)."""
        ne, nl, ns = C.c_uint64(), C.c_uint64(), C.c_uint32()
        self._ck(self.L.chd_get_visible_delta(self.h, None, None, None, None, 0, C.byref(ne), C.byref(nl), C.byref(ns)))
        return ne.value, nl.value, ns.value

    def get_visible_delta(self):
        """-> (enter_off[n+1] u64, enter u32, leave_off[n+1] u64, leave u32), n = slots the delta covers."""
        ne, nl, ns = self.visible_delta_counts()
        eo, lo = np.zeros(ns + 1, np.uint64), np.zeros(ns + 1, np.uint64)
        en, le = np.zeros(max(ne, 1), np.uint32), np.zeros(max(nl, 1), np.uint32)
        self._ck(self.L.chd_get_visible_delta(self.h, ptr(eo), ptr(en), ptr(lo), ptr(le), max(ne, nl, 1), None, None, None))
        return eo, en[:ne], lo, le[:nl]

    # ---- entity-table mode: entities spawned, moved and despawned by id; every result names ids
    def entity_table_init(self):
        self._ck(self.L.chd_entity_table_init(self.h))

    def _events(self, fn, ids, x=None, z=None, dtype=np.float64, status=True):
        # numpy arrays and sequences are converted; torch tensors (pinned host or CUDA) are passed as they are
        if not hasattr(ids, "data_ptr"):
            ids = np.ascontiguousarray(ids, np.uint32)
        if x is not None and not hasattr(x, "data_ptr"):
            x = np.ascontiguousarray(x, dtype)
            z = np.ascontiguousarray(z, dtype)
        n = len(ids)
        args = [self.h, ptr(ids)] + ([] if x is None else [ptr(x), ptr(z)]) + [n]
        if not status:
            self._keep_moves = [ids, x, z]  # the H2D copy is asynchronous: referenced until the next move
            self._ck(fn(*args))
            return None
        st = np.zeros(n, np.uint8)
        self._ck(fn(*(args + [ptr(st)])))
        return st

    def spawn_entities(self, ids, x, z):
        """-> per-event status (capi.EV_*)."""
        return self._events(self.L.chd_spawn_entities, ids, x, z)

    def spawn_entities_f32(self, ids, x, z):
        return self._events(self.L.chd_spawn_entities_f32, ids, x, z, np.float32)

    def despawn_entities(self, ids):
        return self._events(self.L.chd_despawn_entities, ids)

    def move_entities(self, ids, x, z):
        self._events(self.L.chd_move_entities, ids, x, z, status=False)

    def move_entities_f32(self, ids, x, z):
        self._events(self.L.chd_move_entities_f32, ids, x, z, np.float32, status=False)

    # facings (include/chd_gpu_facing.h, entity-table mode): (fx, fz) per id, (cos yaw, sin yaw); (0, 0) or non-finite = none
    def spawn_entities_facing(self, ids, x, z, fx, fz):
        """-> per-event status (capi.EV_*)."""
        return self._facing_events(self.L.chd_spawn_entities_facing, ids, x, z, fx, fz, np.float64, True)

    def spawn_entities_facing_f32(self, ids, x, z, fx, fz):
        return self._facing_events(self.L.chd_spawn_entities_facing_f32, ids, x, z, fx, fz, np.float32, True)

    def move_entities_facing(self, ids, x, z, fx, fz):
        """Position and facing together; the facing of an id's last move in the call wins with its position."""
        self._facing_events(self.L.chd_move_entities_facing, ids, x, z, fx, fz, np.float64, False)

    def move_entities_facing_f32(self, ids, x, z, fx, fz):
        self._facing_events(self.L.chd_move_entities_facing_f32, ids, x, z, fx, fz, np.float32, False)

    def _facing_events(self, fn, ids, x, z, fx, fz, dtype, status):
        arrs = [a if hasattr(a, "data_ptr") else np.ascontiguousarray(a, dt) for a, dt in
                ((ids, np.uint32), (x, dtype), (z, dtype), (fx, dtype), (fz, dtype))]
        n = len(arrs[0])
        if not status:
            self._keep_moves = arrs  # the H2D copy is asynchronous: referenced until the next move
            self._ck(fn(self.h, *(ptr(a) for a in arrs), n))
            return None
        st = np.zeros(n, np.uint8)
        self._ck(fn(self.h, *(ptr(a) for a in arrs), n, ptr(st)))
        return st

    def entity_stats(self):
        s = capi.EntityStats()
        self._ck(self.L.chd_get_entity_stats(self.h, C.byref(s)))
        return s.as_dict()

    # ---- followers: subscriber slots whose AOI is centred on an entity; the device generates the tick's query batch
    def follow_bind(self, slots, entities, kind=None, sph_r=None, box=None, cone=None):
        """Binds slot[i] to entity[i] (entity index; table id in entity-table mode).  kind: AOI_SPHERE | AOI_BOX | AOI_CONE masks
        (None = all sphere); sph_r, box=(ex, ez), cone=(dx, dz, angle, r): per-binding shape arrays of the kinds in use."""
        slots = np.ascontiguousarray(slots, np.uint32)
        entities = np.ascontiguousarray(entities, np.uint32)
        keep = [slots, entities]

        def arr(a, dtype=np.float64):
            if a is None:
                return None
            a = np.ascontiguousarray(a, dtype)
            keep.append(a)
            return ptr(a)

        b = capi.FollowBatch()
        b.n, b.slot, b.entity, b.kind, b.sph_r = len(slots), ptr(slots), ptr(entities), arr(kind, np.uint8), arr(sph_r)
        if box is not None:
            b.box_ex, b.box_ez = (arr(a) for a in box)
        if cone is not None:
            b.cone_dx, b.cone_dz, b.cone_angle, b.cone_r = (arr(a) for a in cone)
        self._ck(self.L.chd_follow_bind(self.h, C.byref(b)))

    def follow_unbind(self, slots):
        slots = np.ascontiguousarray(slots, np.uint32)
        self._ck(self.L.chd_follow_unbind(self.h, ptr(slots), len(slots)))

    def follow_queries(self, mode=capi.FOLLOW_ALL):
        """Generates the tick's query batch from the bindings (asynchronous); the next begin_interest(None) /
        update_interest(None) or tick(None, flags | TICK_FOLLOW) consumes it."""
        self._ck(self.L.chd_follow_queries(self.h, int(mode)))

    def follow_queries_with(self, mode=capi.FOLLOW_ALL, batch=None):
        """follow_queries(mode) with the tick's explicit queries in front: `batch` (a chd_query_batch, sub required), or with
        batch None the batch handed over by prefetch_queries + adopt_prefetched.  The merged batch has host_part_size(n) + followers
        entries; it is consumed like follow_queries' batch."""
        self._ck(self.L.chd_follow_queries_with(self.h, int(mode), C.byref(batch) if batch is not None else None))

    def get_follow(self):
        """-> dict(slot, entity, status, cx, cz: one entry per follower in slot order; n_selected)."""
        n, sel = C.c_uint32(), C.c_uint32()
        self._ck(self.L.chd_get_follow(self.h, None, None, None, None, None, 0, C.byref(n), C.byref(sel)))
        k = n.value
        slot, ent, st = np.zeros(k, np.uint32), np.zeros(k, np.uint32), np.zeros(k, np.uint32)
        cx, cz = np.zeros(k), np.zeros(k)
        if k:
            self._ck(self.L.chd_get_follow(self.h, ptr(slot), ptr(ent), ptr(st), ptr(cx), ptr(cz), k, None, None))
        return dict(slot=slot, entity=ent, status=st, cx=cx, cz=cz, n_selected=sel.value)

    def follow_set_frame(self, slots, off_fwd=None, off_right=None, rot=None):
        """Frames of bound followers (include/chd_gpu_facing.h): centre offsets along / to the right of the entity's facing, and
        rot=(cos, sin) arrays turning the cone relative to the facing (None: the identity)."""
        slots = np.ascontiguousarray(slots, np.uint32)
        n = len(slots)
        keep = [slots]

        def arr(a):
            if a is None:
                return None
            a = np.ascontiguousarray(np.broadcast_to(np.asarray(a, np.float64), (n,)))
            keep.append(a)
            return ptr(a)

        b = capi.FollowFrameBatch(n=n, slot=ptr(slots), off_fwd=arr(off_fwd), off_right=arr(off_right))
        if rot is not None:
            b.rot_cos, b.rot_sin = arr(rot[0]), arr(rot[1])
        self._ck(self.L.chd_follow_set_frame(self.h, C.byref(b)))

    def get_follow_frame(self):
        """-> dict(slot, fx, fz, cx, cz, dx, dz): every framed follower in slot order with the facing, centre and cone direction
        of its last query."""
        n = C.c_uint32()
        self._ck(self.L.chd_get_follow_frame(self.h, None, None, None, None, None, None, None, 0, C.byref(n)))
        k = n.value
        out = dict(slot=np.zeros(k, np.uint32), **{a: np.zeros(k) for a in ("fx", "fz", "cx", "cz", "dx", "dz")})
        if k:
            self._ck(self.L.chd_get_follow_frame(self.h, *(ptr(out[a]) for a in ("slot", "fx", "fz", "cx", "cz", "dx", "dz")), k, C.byref(n)))
        return out

    def device_view(self, which):
        p, n = C.c_void_p(), C.c_uint64()
        self._ck(self.L.chd_device_view(self.h, which, C.byref(p), C.byref(n)))
        return p.value, n.value

    # ---- instrumentation
    def launch_count(self):
        return int(self.L.chd_launch_count(self.h))

    def enable_graphs(self, on=True):
        self._ck(self.L.chd_enable_graphs(self.h, int(bool(on))))

    def graph_launch_count(self):
        return int(self.L.chd_graph_launch_count(self.h))

    def profile_enable(self, on=True):
        """True / 1: every stage; 2: the emit kernel only; False / 0: off."""
        self._ck(self.L.chd_profile_enable(self.h, 2 if on == 2 else int(bool(on))))

    def profile_get(self, stage):
        ms, n = C.c_double(), C.c_uint64()
        self._ck(self.L.chd_profile_get(self.h, int(stage), C.byref(ms), C.byref(n)))
        return ms.value, n.value

    def profile_timeline(self, stage):
        a, b = C.c_double(), C.c_double()
        self._ck(self.L.chd_profile_timeline(self.h, int(stage), C.byref(a), C.byref(b)))
        return a.value, b.value

    # ---- multi-GPU: the NCCL exchange behind the C ABI
    @staticmethod
    def comm_unique_id():
        buf = (C.c_uint8 * 128)()
        st = capi.lib().chd_comm_unique_id(buf)
        if st != capi.OK:
            raise ChdError(st, "chd_comm_unique_id failed (libnccl.so.2 missing?)")
        return bytes(buf)

    def comm_init(self, unique_id, rank, world, halo_cols, border_capacity, migrate_subscribers=0, migrate_pairs=0):
        buf = (C.c_uint8 * 128).from_buffer_copy(bytes(unique_id))
        self._ck(self.L.chd_comm_init(self.h, buf, int(rank), int(world), int(halo_cols), int(border_capacity), int(migrate_subscribers),
                                      int(migrate_pairs)))

    def migrate_out(self, slots):
        slots = np.ascontiguousarray(slots, np.uint32)
        self._ck(self.L.chd_migrate_out(self.h, ptr(slots), len(slots)))

    def migrate_in(self, src_rank, first_index, slots, conn_ids):
        slots = np.ascontiguousarray(slots, np.uint32)
        conn_ids = np.ascontiguousarray(conn_ids, np.uint32)
        self._ck(self.L.chd_migrate_in(self.h, int(src_rank), int(first_index), ptr(slots), ptr(conn_ids), len(slots)))
        if len(slots):
            self.n_slots = max(self.n_slots, int(slots.max()) + 1)

    def get_rehome(self, cap=1 << 20):
        gid, dst, n = np.zeros(cap, np.uint32), np.zeros(cap, np.uint32), C.c_uint32()
        self._ck(self.L.chd_get_rehome(self.h, ptr(gid), ptr(dst), cap, C.byref(n)))
        k = min(n.value, cap)
        return gid[:k].copy(), dst[:k].copy(), n.value

    def handoff_entities(self, cap=1 << 16):
        """Entity-table mode on slabs: lists the own entities whose column another rank owns and removes them from this table
        -> (id u32, dst_rank u32, x f64, z f64); the receiving rank adopts them with spawn_entities(id, x, z)."""
        n = C.c_uint32()
        while True:
            ids, dst, x, z = np.zeros(cap, np.uint32), np.zeros(cap, np.uint32), np.zeros(cap), np.zeros(cap)
            st = self.L.chd_handoff_entities(self.h, ptr(ids), ptr(dst), ptr(x), ptr(z), int(cap), C.byref(n))
            if st != capi.ERR_CAPACITY or n.value <= cap:
                break
            cap = n.value  # nothing was removed: the same list again, with room for it
        self._ck(st)
        k = n.value
        return ids[:k].copy(), dst[:k].copy(), x[:k].copy(), z[:k].copy()

    def handoff_entities_facing(self, cap=1 << 16):
        """handoff_entities with each entity's facing -> (id, dst_rank, x, z, fx, fz); the receiving rank adopts them with
        spawn_entities_facing(id, x, z, fx, fz)."""
        n = C.c_uint32()
        while True:
            ids, dst = np.zeros(cap, np.uint32), np.zeros(cap, np.uint32)
            x, z, fx, fz = np.zeros(cap), np.zeros(cap), np.zeros(cap), np.zeros(cap)
            st = self.L.chd_handoff_entities_facing(self.h, ptr(ids), ptr(dst), ptr(x), ptr(z), ptr(fx), ptr(fz), int(cap), C.byref(n))
            if st != capi.ERR_CAPACITY or n.value <= cap:
                break
            cap = n.value
        self._ck(st)
        k = n.value
        return ids[:k].copy(), dst[:k].copy(), x[:k].copy(), z[:k].copy(), fx[:k].copy(), fz[:k].copy()

    def comm_info(self):
        r, w, ver = C.c_int(), C.c_int(), C.c_int()
        lo, hi, halo = C.c_uint32(), C.c_uint32(), C.c_uint32()
        self._ck(self.L.chd_comm_info(self.h, C.byref(r), C.byref(w), C.byref(lo), C.byref(hi), C.byref(halo), C.byref(ver)))
        return dict(rank=r.value, world=w.value, col_lo=lo.value, col_hi=hi.value, halo=halo.value, nccl_version=ver.value)

    def tick_sharded(self, batch, t_ns, flags=capi.TICK_ALL, want_summary=True):
        s = TickSummary() if want_summary else None
        self._ck(self.L.chd_tick_sharded(self.h, C.byref(batch) if batch is not None else None, int(t_ns), int(flags),
                                         C.byref(s) if s is not None else None))
        return s

    def collective_count(self):
        return int(self.L.chd_collective_count(self.h))

    def exchange_mode(self):
        """0 no communicator, 1 ncclAllGather per tick, 2 peer windows (stores over NVLink + flags, no collective on the tick path)."""
        return int(self.L.chd_comm_exchange_mode(self.h))

    def use_collective(self, on=True):
        self._ck(self.L.chd_comm_use_collective(self.h, 1 if on else 0))

    # ---- multi-GPU slab
    def set_slab(self, col_lo, col_hi, halo):
        self._ck(self.L.chd_set_slab(self.h, int(col_lo), int(col_hi), int(halo)))

    def export_border(self, d_records, cap_records, want_count=True):
        """want_count=False keeps the call free of host synchronisation (overflow shows up in the next summary)."""
        if not want_count:
            self._ck(self.L.chd_export_border(self.h, ptr(d_records), int(cap_records), None))
            return None
        n = C.c_uint32()
        self._ck(self.L.chd_export_border(self.h, ptr(d_records), int(cap_records), C.byref(n)))
        return n.value

    def import_halo(self, d_records, n_records, skip_first, skip_count):
        self._ck(self.L.chd_import_halo(self.h, ptr(d_records), int(n_records), int(skip_first), int(skip_count)))

    # ---- ring limits across slabs (include/chd_gpu_rings.h): device record buffers, 2 x u32 (cell, maxFanOutIntervalMs) each
    def export_ring_limits(self, d_records, cap, want_count=True):
        """Records of the served cells whose limit rose since their last export or import -> their count (None with
        want_count=False: no host synchronisation, an overflow shows up in the next summary)."""
        if not want_count:
            self._ck(self.L.chd_export_ring_limits(self.h, ptr(d_records), int(cap), None))
            return None
        n = C.c_uint32()
        self._ck(self.L.chd_export_ring_limits(self.h, ptr(d_records), int(cap), C.byref(n)))
        return n.value

    def import_ring_limits(self, d_records, n):
        self._ck(self.L.chd_import_ring_limits(self.h, ptr(d_records), int(n)))

    # ---- byte-carrying device rings (include/chd_gpu_ring_bytes.h)
    def rings_reserve_bytes(self, bytes_per_cell):
        """After chd_rings_init and before any append: every ring entry carries its update's serialized bytes, in a slab of
        bytes_per_cell bytes per cell."""
        self._ck(self.L.chd_rings_reserve_bytes(self.h, int(bytes_per_cell)))

    def rings_append_bytes(self, upd_off, arrival, sender, byte_off, data):
        """chd_rings_append with update k carrying data[byte_off[k]:byte_off[k + 1]] (byte_off: host u64, n_updates + 1 offsets;
        data: bytes, a u8 array or a device tensor)."""
        upd_off = np.ascontiguousarray(upd_off, np.uint32)
        arrival = np.ascontiguousarray(arrival, np.int64)
        sender = np.ascontiguousarray(sender, np.uint32)
        byte_off = np.ascontiguousarray(byte_off, np.uint64)
        if isinstance(data, (bytes, bytearray)):
            data = np.frombuffer(data, np.uint8)
        n = len(byte_off) - 1
        self._ck(self.L.chd_rings_append_bytes(self.h, ptr(upd_off), n, ptr(arrival) if n else None, ptr(sender) if n else None, ptr(byte_off),
                                               ptr(data) if len(data) else None))

    def get_ring_bytes(self):
        """-> (byte_off u64 [n_live + 1], data u8): every live ring entry's bytes, in the entry order of get_rings"""
        off = self._ring_off()
        total = C.c_uint64()
        self._ck(self.L.chd_get_ring_bytes(self.h, None, None, 0, C.byref(total)))
        byte_off, data = np.zeros(int(off[-1]) + 1, np.uint64), np.zeros(total.value + 1, np.uint8)
        self._ck(self.L.chd_get_ring_bytes(self.h, ptr(byte_off), ptr(data), total.value, C.byref(total)))
        return byte_off, data[:total.value]
