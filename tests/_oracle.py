"""ctypes binding of the CPU oracle (oracle/libchd_oracle.so).  Test infrastructure only:
nothing under channeld_b200/ may import this module."""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")

u32p = C.POINTER(C.c_uint32)
u64p = C.POINTER(C.c_uint64)
f64p = C.POINTER(C.c_double)

AOI_SPOTS, AOI_BOX, AOI_SPHERE, AOI_CONE = 1, 2, 4, 8
OK, ERR_OUT_OF_WORLD, ERR_BAD_STEP, ERR_NIL, ERR_CAPACITY, ERR_ITER = 0, 1, 2, 3, 4, 5


class Grid(C.Structure):
    _fields_ = [
        ("world_offset_x", C.c_double), ("world_offset_z", C.c_double),
        ("grid_width", C.c_double), ("grid_height", C.c_double),
        ("grid_cols", C.c_uint32), ("grid_rows", C.c_uint32),
        ("server_cols", C.c_uint32), ("server_rows", C.c_uint32),
        ("server_interest_border_size", C.c_uint32), ("channel_id_start", C.c_uint32),
    ]


class Query(C.Structure):
    _fields_ = [
        ("kind_mask", C.c_uint32), ("n_spots", C.c_uint32), ("n_spot_dists", C.c_uint32),
        ("spot_x", f64p), ("spot_z", f64p), ("spot_dist", u32p),
        ("box_cx", C.c_double), ("box_cz", C.c_double), ("box_ex", C.c_double), ("box_ez", C.c_double),
        ("sph_cx", C.c_double), ("sph_cz", C.c_double), ("sph_r", C.c_double),
        ("cone_cx", C.c_double), ("cone_cz", C.c_double), ("cone_dx", C.c_double), ("cone_dz", C.c_double),
        ("cone_angle", C.c_double), ("cone_r", C.c_double),
    ]


class QuerySoA(C.Structure):
    _fields_ = [("n", C.c_uint32), ("kind", C.c_void_p)] + [(k, f64p) for k in (
        "sph_cx", "sph_cz", "sph_r", "box_cx", "box_cz", "box_ex", "box_ez", "cone_cx", "cone_cz", "cone_dx", "cone_dz", "cone_angle",
        "cone_r")] + [("spot_off", u32p), ("spot_ndist", u32p), ("spot_x", f64p), ("spot_z", f64p), ("spot_dist", u32p)]


class Send(C.Structure):
    _fields_ = [
        ("conn_id", C.c_uint32), ("kind", C.c_uint32), ("n_selected", C.c_uint32),
        ("first_sel", C.c_uint32), ("last_sel", C.c_uint32), ("sel_hash", C.c_uint64),
        ("last_message_index", C.c_uint64), ("window_hi", C.c_int64),
    ]


def make_grid(offx, offz, w, h, cols, rows, scols=1, srows=1, border=0, id_start=0x10000):
    return Grid(float(offx), float(offz), float(w), float(h), cols, rows, scols, srows, border, id_start)


def _p(a, t):
    return a.ctypes.data_as(t)


class Oracle:
    def __init__(self, lib):
        self.lib = lib
        L = lib
        L.orc_grid_size.restype = C.c_double
        L.orc_grid_size.argtypes = [C.POINTER(Grid)]
        L.orc_go_cos.restype = C.c_double
        L.orc_go_cos.argtypes = [C.c_double]
        L.orc_get_channel_id.restype = C.c_int
        L.orc_get_channel_id.argtypes = [C.POINTER(Grid), C.c_double, C.c_double, u32p]
        L.orc_cell_of.restype = None
        L.orc_cell_of.argtypes = [C.POINTER(Grid), f64p, f64p, C.c_uint32, u32p]
        L.orc_query_channel_ids.restype = C.c_int
        L.orc_query_channel_ids.argtypes = [C.POINTER(Grid), C.POINTER(Query), u32p, u32p, C.c_uint32, u32p]
        L.orc_query_batch.restype = C.c_int
        L.orc_query_batch.argtypes = [C.POINTER(Grid), C.POINTER(QuerySoA), u32p, u64p, u32p, u32p, C.c_uint64, C.c_int]
        L.orc_get_adjacent_channels.restype = C.c_uint32
        L.orc_get_adjacent_channels.argtypes = [C.POINTER(Grid), C.c_uint32, u32p]
        L.orc_adjacent_broadcast.restype = C.c_uint32
        L.orc_adjacent_broadcast.argtypes = [C.POINTER(Grid), C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, u32p, u32p, C.c_void_p, u32p, C.c_uint32]
        L.orc_get_regions.restype = None
        L.orc_get_regions.argtypes = [C.POINTER(Grid), f64p, f64p, f64p, f64p, u32p, u32p]
        L.orc_damping_interval_ms.restype = C.c_uint32
        L.orc_damping_interval_ms.argtypes = [C.c_uint32, C.c_uint32]
        L.orc_interest_diff.restype = None
        L.orc_interest_diff.argtypes = [u32p, C.c_uint32, u32p, C.c_uint32, u32p, u32p, u32p, u32p, u32p, u32p]
        L.orc_channel_new.restype = C.c_void_p
        L.orc_channel_free.argtypes = [C.c_void_p]
        L.orc_channel_subscribe.restype = C.c_int
        L.orc_channel_subscribe.argtypes = [C.c_void_p, C.c_uint32, C.c_int64, C.c_uint32, C.c_int32, C.c_int, C.c_int]
        L.orc_channel_unsubscribe.restype = C.c_int
        L.orc_channel_unsubscribe.argtypes = [C.c_void_p, C.c_uint32]
        L.orc_channel_on_update.restype = None
        L.orc_channel_on_update.argtypes = [C.c_void_p, C.c_int64, C.c_uint32]
        L.orc_channel_ring_len.restype = C.c_uint32
        L.orc_channel_ring_len.argtypes = [C.c_void_p]
        L.orc_channel_tick_data_ex.restype = C.c_uint32
        L.orc_channel_tick_data_ex.argtypes = [C.c_void_p, C.c_int64, C.POINTER(Send), C.c_uint32, C.POINTER(C.c_int64), u32p, u32p, u32p, C.c_uint32]
        L.orc_channel_tick_data.restype = C.c_uint32
        L.orc_channel_tick_data.argtypes = [C.c_void_p, C.c_int64, C.POINTER(Send), C.c_uint32]
        L.orc_channel_get_state.restype = C.c_int
        L.orc_channel_get_state.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_int64), C.POINTER(C.c_int), u64p]
        vp = C.c_void_p
        L.orc_channels_subscribe.restype = None
        L.orc_channels_subscribe.argtypes = [vp, u32p, u32p, u32p, C.c_uint64, C.c_int64, C.c_int32, C.c_int, C.c_int]
        L.orc_channels_unsubscribe.restype = None
        L.orc_channels_unsubscribe.argtypes = [vp, u32p, u32p, C.c_uint64]
        L.orc_channels_on_update.restype = None
        L.orc_channels_on_update.argtypes = [vp, u32p, C.POINTER(C.c_int64), u32p, C.c_uint64]
        L.orc_channels_tick_data.restype = C.c_uint64
        L.orc_channels_tick_data.argtypes = [vp, C.c_uint32, C.c_int64, C.POINTER(Send), C.c_uint64, u64p]
        L.orc_channels_tick_data_ex.restype = C.c_uint64
        L.orc_channels_tick_data_ex.argtypes = [vp, C.c_uint32, C.c_int64, C.POINTER(Send), C.c_uint64, u64p, C.POINTER(C.c_int64), u32p, u64p,
                                                u32p, C.c_uint64]
        L.orc_channels_get_rings.restype = C.c_uint64
        L.orc_channels_get_rings.argtypes = [vp, C.c_uint32, u64p, C.POINTER(C.c_int64), u32p, u64p, C.c_uint64, u64p, u32p]
        L.orc_channels_get_state.restype = None
        L.orc_channels_get_state.argtypes = [vp, u32p, u32p, C.c_uint64, C.POINTER(C.c_int64), C.POINTER(C.c_uint8), u64p,
                                             C.POINTER(C.c_uint8)]
        L.orc_sphere_tick.restype = C.c_int
        L.orc_sphere_tick.argtypes = [C.POINTER(Grid), f64p, f64p, C.c_uint32, f64p, f64p, f64p, C.c_uint32,
                                      u32p, u64p, u32p, u32p, C.c_uint64, u64p, u32p, C.c_uint64, C.c_int]
        L.orc_visible_delta.restype = C.c_int
        L.orc_visible_delta.argtypes = [C.c_uint32, u32p, C.c_uint32, u64p, u32p, C.c_uint32, u32p, C.c_uint32, u64p, u32p, C.c_uint32,
                                        u64p, u32p, C.c_uint64, u64p, u32p, C.c_uint64, C.c_int]
        L.orc_baseline_run.restype = C.c_uint64
        L.orc_baseline_run.argtypes = [C.POINTER(Grid), f64p, f64p, C.c_uint32, f64p, f64p, f64p,
                                       C.c_uint32, C.c_uint32, C.c_int, C.c_int]

    # ---- spatial.go ----
    def grid_size(self, g):
        return self.lib.orc_grid_size(C.byref(g))

    def go_cos(self, x):
        return self.lib.orc_go_cos(float(x))

    def get_channel_id(self, g, x, z):
        """-> (id, err) like StaticGrid2DSpatialController.GetChannelId"""
        out = C.c_uint32(0)
        st = self.lib.orc_get_channel_id(C.byref(g), float(x), float(z), C.byref(out))
        return out.value, st

    def cell_of(self, g, x, z):
        x = np.ascontiguousarray(x, np.float64)
        z = np.ascontiguousarray(z, np.float64)
        out = np.zeros(len(x), np.uint32)
        self.lib.orc_cell_of(C.byref(g), _p(x, f64p), _p(z, f64p), len(x), _p(out, u32p))
        return out

    def query(self, g, *, spots=None, spot_dists=None, box=None, sphere=None, cone=None, cap=1 << 20):
        """-> (dict{channel_id: dist} | None, status).  box=(cx,cz,ex,ez) sphere=(cx,cz,r)
        cone=(cx,cz,dx,dz,angle,r) spots=[(x,z),...]"""
        q = Query()
        keep = []
        if spots is not None:
            q.kind_mask |= AOI_SPOTS
            sx = np.array([s[0] for s in spots], np.float64)
            sz = np.array([s[1] for s in spots], np.float64)
            sd = np.array(spot_dists if spot_dists is not None else [], np.uint32)
            keep += [sx, sz, sd]
            q.n_spots, q.n_spot_dists = len(sx), len(sd)
            q.spot_x, q.spot_z, q.spot_dist = _p(sx, f64p), _p(sz, f64p), _p(sd, u32p)
        if box is not None:
            q.kind_mask |= AOI_BOX
            q.box_cx, q.box_cz, q.box_ex, q.box_ez = map(float, box)
        if sphere is not None:
            q.kind_mask |= AOI_SPHERE
            q.sph_cx, q.sph_cz, q.sph_r = map(float, sphere)
        if cone is not None:
            q.kind_mask |= AOI_CONE
            q.cone_cx, q.cone_cz, q.cone_dx, q.cone_dz, q.cone_angle, q.cone_r = map(float, cone)
        ids = np.zeros(cap, np.uint32)
        dists = np.zeros(cap, np.uint32)
        n = C.c_uint32(0)
        st = self.lib.orc_query_channel_ids(C.byref(g), C.byref(q), _p(ids, u32p), _p(dists, u32p), cap, C.byref(n))
        if st != OK:
            return None, st
        return {int(ids[i]): int(dists[i]) for i in range(n.value)}, st

    def query_batch(self, g, n, kind=None, sphere=None, box=None, cone=None, spots=None, n_threads=None):
        """orc_query_batch on a batch in engine.make_batch's form: kind[n] masks (None = all sphere), sphere=(cx,cz,r)
        box=(cx,cz,ex,ez) cone=(cx,cz,dx,dz,angle,r) tuples of arrays, spots=(spot_off, spot_ndist, x, z, dist).
        -> (status u32[n], off u64[n+1], channel_id u32[], dist u32[])"""
        b = QuerySoA()
        b.n = int(n)
        keep = []

        def arr(a, dt, t):
            a = np.ascontiguousarray(a, dt)
            keep.append(a)
            return _p(a, t)

        if kind is not None:
            k = np.ascontiguousarray(kind, np.uint8)
            keep.append(k)
            b.kind = k.ctypes.data
        for names, vals in ((("sph_cx", "sph_cz", "sph_r"), sphere), (("box_cx", "box_cz", "box_ex", "box_ez"), box),
                            (("cone_cx", "cone_cz", "cone_dx", "cone_dz", "cone_angle", "cone_r"), cone)):
            if vals is not None:
                for name, v in zip(names, vals):
                    setattr(b, name, arr(v, np.float64, f64p))
        if spots is not None:
            off, ndist, x, z, dist = spots
            b.spot_off, b.spot_x, b.spot_z = arr(off, np.uint32, u32p), arr(x, np.float64, f64p), arr(z, np.float64, f64p)
            if ndist is not None:
                b.spot_ndist = arr(ndist, np.uint32, u32p)
            if dist is not None:
                b.spot_dist = arr(dist, np.uint32, u32p)
        status = np.zeros(max(n, 1), np.uint32)
        off = np.zeros(n + 1, np.uint64)
        nt = int(n_threads or os.cpu_count() or 1)
        cap = 64 * n + 1024
        while True:
            ids, dist = np.zeros(cap, np.uint32), np.zeros(cap, np.uint32)
            rc = self.lib.orc_query_batch(C.byref(g), C.byref(b), _p(status, u32p), _p(off, u64p), _p(ids, u32p), _p(dist, u32p), cap, nt)
            if rc != ERR_CAPACITY:
                break
            cap = int(off[n])
        assert rc == OK, rc
        t = int(off[n])
        return status[:n], off, ids[:t], dist[:t]

    def adjacent(self, g, channel_id):
        out = np.zeros(8, np.uint32)
        n = self.lib.orc_get_adjacent_channels(C.byref(g), channel_id, _p(out, u32p))
        return [int(v) for v in out[:n]]

    def adjacent_broadcast(self, g, channel_id, broadcast, sender, client, cell_off, conn_id, conn_type):
        """message.go:188-239 on per-cell subscriber lists (CSR) -> sorted recipient connection ids."""
        cell_off = np.ascontiguousarray(cell_off, np.uint32)
        conn_id = np.ascontiguousarray(conn_id, np.uint32)
        ct = None if conn_type is None else np.ascontiguousarray(conn_type, np.uint8)
        cap = len(conn_id) + 1
        out = np.zeros(cap, np.uint32)
        n = self.lib.orc_adjacent_broadcast(C.byref(g), int(channel_id), int(broadcast), int(sender), int(client), _p(cell_off, u32p),
                                            _p(conn_id, u32p), None if ct is None else ct.ctypes.data_as(C.c_void_p), _p(out, u32p), cap)
        return out[:n].copy()

    def regions(self, g):
        n = g.grid_cols * g.grid_rows
        a = [np.zeros(n, np.float64) for _ in range(4)]
        cid = np.zeros(n, np.uint32)
        srv = np.zeros(n, np.uint32)
        self.lib.orc_get_regions(C.byref(g), *[_p(v, f64p) for v in a], _p(cid, u32p), _p(srv, u32p))
        return a[0], a[1], a[2], a[3], cid, srv

    def damping(self, dist, default_ms=20):
        return self.lib.orc_damping_interval_ms(dist, default_ms)

    def interest_diff(self, existing, wanted):
        ex = np.ascontiguousarray(existing, np.uint32)
        wa = np.ascontiguousarray(wanted, np.uint32)
        un = np.zeros(max(len(ex), 1), np.uint32)
        sn = np.zeros(max(len(wa), 1), np.uint32)
        kp = np.zeros(max(len(wa), 1), np.uint32)
        nu, ns, nk = C.c_uint32(0), C.c_uint32(0), C.c_uint32(0)
        self.lib.orc_interest_diff(_p(ex, u32p), len(ex), _p(wa, u32p), len(wa), _p(un, u32p), C.byref(nu),
                                   _p(sn, u32p), C.byref(ns), _p(kp, u32p), C.byref(nk))
        return un[:nu.value].copy(), sn[:ns.value].copy(), kp[:nk.value].copy()

    # ---- data.go ----
    def channel(self):
        return OracleChannel(self)

    def channels(self, n):
        return OracleChannels(self, n)

    # ---- derived ----
    def sphere_tick(self, g, ex, ez, cx, cz, r):
        ex = np.ascontiguousarray(ex, np.float64); ez = np.ascontiguousarray(ez, np.float64)
        cx = np.ascontiguousarray(cx, np.float64); cz = np.ascontiguousarray(cz, np.float64)
        r = np.ascontiguousarray(r, np.float64)
        nq = len(cx)
        status = np.zeros(nq, np.uint32)
        poff = np.zeros(nq + 1, np.uint64)
        voff = np.zeros(nq + 1, np.uint64)
        self.lib.orc_sphere_tick(C.byref(g), _p(ex, f64p), _p(ez, f64p), len(ex), _p(cx, f64p), _p(cz, f64p),
                                 _p(r, f64p), nq, _p(status, u32p), _p(poff, u64p), None, None, 0,
                                 _p(voff, u64p), None, 0, 1)
        P, V = int(poff[nq]), int(voff[nq])
        pc = np.zeros(max(P, 1), np.uint32); pd = np.zeros(max(P, 1), np.uint32)
        ve = np.zeros(max(V, 1), np.uint32)
        rc = self.lib.orc_sphere_tick(C.byref(g), _p(ex, f64p), _p(ez, f64p), len(ex), _p(cx, f64p), _p(cz, f64p),
                                      _p(r, f64p), nq, _p(status, u32p), _p(poff, u64p), _p(pc, u32p), _p(pd, u32p), P,
                                      _p(voff, u64p), _p(ve, u32p), V, 1)
        assert rc == 0
        return dict(status=status, pair_off=poff, pair_cell=pc[:P], pair_dist=pd[:P], vis_off=voff, vis_entity=ve[:V])

    def sphere_pairs(self, g, ex, ez, cx, cz, r):
        """sphere_tick without the visible lists (only their offsets): -> dict(status, pair_off u64, pair_cell channel ids, pair_dist,
        vis_off)"""
        ex = np.ascontiguousarray(ex, np.float64); ez = np.ascontiguousarray(ez, np.float64)
        cx = np.ascontiguousarray(cx, np.float64); cz = np.ascontiguousarray(cz, np.float64)
        r = np.ascontiguousarray(r, np.float64)
        nq = len(cx)
        status = np.zeros(nq, np.uint32)
        poff = np.zeros(nq + 1, np.uint64)
        voff = np.zeros(nq + 1, np.uint64)
        args = (C.byref(g), _p(ex, f64p), _p(ez, f64p), len(ex), _p(cx, f64p), _p(cz, f64p), _p(r, f64p), nq, _p(status, u32p), _p(poff, u64p))
        self.lib.orc_sphere_tick(*args, None, None, 0, _p(voff, u64p), None, 0, 1)
        P = int(poff[nq])
        pc = np.zeros(max(P, 1), np.uint32); pd = np.zeros(max(P, 1), np.uint32)
        rc = self.lib.orc_sphere_tick(*args, _p(pc, u32p), _p(pd, u32p), P, _p(voff, u64p), None, 0, 1)
        assert rc == 0
        return dict(status=status, pair_off=poff, pair_cell=pc[:P], pair_dist=pd[:P], vis_off=voff)

    def visible_delta(self, cells, prev, now, n_threads=None):
        """orc_visible_delta.  prev / now = (cell per entity, pair_off, pair_cell): cells >= `cells` are out of the world, pair cells
        are cell indices.  -> (enter_off u64, enter u32, leave_off u64, leave u32) over max(slots before, slots now) slots."""
        def state(s):
            cell, off, pc = s
            return (np.ascontiguousarray(cell, np.uint32), np.ascontiguousarray(off, np.uint64), np.ascontiguousarray(pc, np.uint32))

        (pcl, poff, ppc), (ncl, noff, npc) = state(prev), state(now)
        n_out = max(len(poff), len(noff)) - 1
        eo, lo = np.zeros(n_out + 1, np.uint64), np.zeros(n_out + 1, np.uint64)
        nt = int(n_threads or os.cpu_count() or 1)
        args = (int(cells), _p(pcl, u32p), len(pcl), _p(poff, u64p), _p(ppc, u32p), len(poff) - 1, _p(ncl, u32p), len(ncl), _p(noff, u64p),
                _p(npc, u32p), len(noff) - 1)
        assert self.lib.orc_visible_delta(*args, _p(eo, u64p), None, 0, _p(lo, u64p), None, 0, nt) == OK
        ne, nl = int(eo[-1]), int(lo[-1])
        en, le = np.zeros(max(ne, 1), np.uint32), np.zeros(max(nl, 1), np.uint32)
        assert self.lib.orc_visible_delta(*args, _p(eo, u64p), _p(en, u32p), ne, _p(lo, u64p), _p(le, u32p), nl, nt) == OK
        return eo, en[:ne], lo, le[:nl]

    def baseline_run(self, g, ex, ez, cx, cz, r, q_begin, q_end, n_threads, build):
        return self.lib.orc_baseline_run(C.byref(g), _p(ex, f64p), _p(ez, f64p), len(ex), _p(cx, f64p), _p(cz, f64p),
                                         _p(r, f64p), q_begin, q_end, n_threads, int(build))


class OracleChannel:
    def __init__(self, orc):
        self.L = orc.lib
        self.h = C.c_void_p(self.L.orc_channel_new())

    def __del__(self):
        try:
            self.L.orc_channel_free(self.h)
        except Exception:
            pass

    def subscribe(self, conn, now_ns, interval_ms, delay_ms=0, skip_self=True, skip_first=False):
        return self.L.orc_channel_subscribe(self.h, conn, int(now_ns), interval_ms, delay_ms, int(skip_self), int(skip_first))

    def unsubscribe(self, conn):
        return self.L.orc_channel_unsubscribe(self.h, conn)

    def on_update(self, arrival_ns, sender):
        self.L.orc_channel_on_update(self.h, int(arrival_ns), sender)

    def ring_len(self):
        return self.L.orc_channel_ring_len(self.h)

    def tick_data(self, t_ns, cap=4096):
        buf = (Send * cap)()
        n = self.L.orc_channel_tick_data(self.h, int(t_ns), buf, cap)
        assert n != 0xFFFFFFFF, "oracle tick_data: capacity/iteration bound"
        return [dict(conn=b.conn_id, kind=b.kind, n=b.n_selected, first=b.first_sel, last=b.last_sel,
                     hash=b.sel_hash, last_index=b.last_message_index, window_hi=b.window_hi) for b in buf[:n]]

    def tick_data_ex(self, t_ns, cap=4096, sel_cap=1 << 18):
        """tick_data + per send: window_lo, self_skipped, and the exact ring positions merged (tuple)."""
        buf = (Send * cap)()
        lo = np.zeros(cap, np.int64)
        sk = np.zeros(cap, np.uint32)
        so = np.zeros(cap + 1, np.uint32)
        sp = np.zeros(sel_cap, np.uint32)
        n = self.L.orc_channel_tick_data_ex(self.h, int(t_ns), buf, cap, lo.ctypes.data_as(C.POINTER(C.c_int64)), _p(sk, u32p), _p(so, u32p),
                                            _p(sp, u32p), sel_cap)
        assert n != 0xFFFFFFFF, "oracle tick_data_ex: capacity/iteration bound"
        return [dict(conn=b.conn_id, kind=b.kind, n=b.n_selected, first=b.first_sel, last=b.last_sel, hash=b.sel_hash,
                     last_index=b.last_message_index, window_hi=b.window_hi, window_lo=int(lo[i]), self_skipped=int(sk[i]),
                     selected=tuple(sp[so[i]:so[i + 1]].tolist())) for i, b in enumerate(buf[:n])]

    def state(self, conn):
        a, b, c = C.c_int64(0), C.c_int(0), C.c_uint64(0)
        rc = self.L.orc_channel_get_state(self.h, conn, C.byref(a), C.byref(b), C.byref(c))
        return None if rc else (a.value, bool(b.value), c.value)


SEND_DTYPE = np.dtype([("conn_id", np.uint32), ("kind", np.uint32), ("n_selected", np.uint32), ("first_sel", np.uint32),
                       ("last_sel", np.uint32), ("sel_hash", np.uint64), ("last_message_index", np.uint64), ("window_hi", np.int64)],
                      align=True)
assert SEND_DTYPE.itemsize == C.sizeof(Send)


class OracleChannels:
    """n oracle channels (one per cell) driven with arrays: the batched orc_channels_* calls, each a loop over the per-channel
    functions OracleChannel wraps."""

    def __init__(self, orc, n):
        self.L = orc.lib
        self.n = n
        self.h = np.array([self.L.orc_channel_new() for _ in range(n)], np.uint64)

    def __del__(self):
        if getattr(self, "_owner", None) is not None:
            return  # a view: its owner frees the channels
        try:
            for h in self.h:
                self.L.orc_channel_free(C.c_void_p(int(h)))
        except Exception:
            pass

    def _hp(self):
        return C.c_void_p(self.h.ctypes.data)

    def subscribe(self, chan, conn, now_ns, interval_ms, delay_ms=0, skip_self=True, skip_first=False):
        chan, conn, iv = (np.ascontiguousarray(a, np.uint32) for a in (chan, conn, interval_ms))
        self.L.orc_channels_subscribe(self._hp(), _p(chan, u32p), _p(conn, u32p), _p(iv, u32p), len(chan), int(now_ns), delay_ms,
                                      int(skip_self), int(skip_first))

    def unsubscribe(self, chan, conn):
        chan, conn = (np.ascontiguousarray(a, np.uint32) for a in (chan, conn))
        self.L.orc_channels_unsubscribe(self._hp(), _p(chan, u32p), _p(conn, u32p), len(chan))

    def on_update(self, chan, arrival_ns, sender):
        chan, sender = (np.ascontiguousarray(a, np.uint32) for a in (chan, sender))
        arrival_ns = np.ascontiguousarray(arrival_ns, np.int64)
        self.L.orc_channels_on_update(self._hp(), _p(chan, u32p), arrival_ns.ctypes.data_as(C.POINTER(C.c_int64)), _p(sender, u32p),
                                      len(chan))

    def tick_data(self, t_ns, cap):
        """-> (sends[SEND_DTYPE], off[n+1]): the sends of channel c are sends[off[c]:off[c+1]]"""
        out = np.zeros(max(int(cap), 1), SEND_DTYPE)
        off = np.zeros(self.n + 1, np.uint64)
        k = self.L.orc_channels_tick_data(self._hp(), self.n, int(t_ns), out.ctypes.data_as(C.POINTER(Send)), int(cap), _p(off, u64p))
        assert k != 2 ** 64 - 1, "oracle tick_data: capacity/iteration bound"
        return out[:k], off

    def tick_data_ex(self, t_ns, cap, sel_cap):
        """tick_data + per send its window_lo, self_skipped and the ring positions merged (positions within its channel's ring)
        -> (sends, off[n+1], window_lo, self_skipped, sel_off u64[len(sends)+1], sel_pos): send i merged sel_pos[sel_off[i]:sel_off[i+1]]"""
        cap = max(int(cap), 1)
        out = np.zeros(cap, SEND_DTYPE)
        off = np.zeros(self.n + 1, np.uint64)
        lo = np.zeros(cap, np.int64)
        sk = np.zeros(cap, np.uint32)
        so = np.zeros(cap + 1, np.uint64)
        sp = np.zeros(max(int(sel_cap), 1), np.uint32)
        k = self.L.orc_channels_tick_data_ex(self._hp(), self.n, int(t_ns), out.ctypes.data_as(C.POINTER(Send)), cap, _p(off, u64p),
                                             lo.ctypes.data_as(C.POINTER(C.c_int64)), _p(sk, u32p), _p(so, u64p), _p(sp, u32p), len(sp))
        assert k != 2 ** 64 - 1, "oracle tick_data_ex: capacity/iteration bound"
        return out[:k], off, lo[:k], sk[:k], so[:k + 1], sp[:int(so[k])]

    def get_rings(self):
        """Every channel's updateMsgBuffer as a CSR by channel -> dict(off u64[n+1], arrival, sender, index (insertion order per
        channel), msg_index u64[n] (ChannelData.msgIndex), max_interval_ms u32[n] (ChannelData.maxFanOutIntervalMs))"""
        off = np.zeros(self.n + 1, np.uint64)
        mi = np.zeros(self.n, np.uint64)
        mx = np.zeros(self.n, np.uint32)
        total = int(self.L.orc_channels_get_rings(self._hp(), self.n, _p(off, u64p), None, None, None, 0, _p(mi, u64p), _p(mx, u32p)))
        arr, snd, idx = np.zeros(max(total, 1), np.int64), np.zeros(max(total, 1), np.uint32), np.zeros(max(total, 1), np.uint64)
        k = self.L.orc_channels_get_rings(self._hp(), self.n, _p(off, u64p), arr.ctypes.data_as(C.POINTER(C.c_int64)), _p(snd, u32p),
                                          _p(idx, u64p), total, None, None)
        assert k == total
        return dict(off=off, arrival=arr[:total], sender=snd[:total], index=idx[:total], msg_index=mi, max_interval_ms=mx)

    def view(self, chans):
        """The channels chans (indices into this set) as a set of their own (the same handles: calls on the view change them)."""
        v = OracleChannels.__new__(OracleChannels)
        v.L, v.h, v.n, v._owner = self.L, np.ascontiguousarray(self.h[np.asarray(chans, np.int64)]), len(chans), self
        return v

    def state(self, chan, conn):
        """-> (last[n], had_first[n], last_index[n], found[n])"""
        chan, conn = (np.ascontiguousarray(a, np.uint32) for a in (chan, conn))
        n = len(chan)
        last = np.zeros(n, np.int64); had = np.zeros(n, np.uint8); li = np.zeros(n, np.uint64); found = np.zeros(n, np.uint8)
        self.L.orc_channels_get_state(self._hp(), _p(chan, u32p), _p(conn, u32p), n, last.ctypes.data_as(C.POINTER(C.c_int64)),
                                      had.ctypes.data_as(C.POINTER(C.c_uint8)), _p(li, u64p), found.ctypes.data_as(C.POINTER(C.c_uint8)))
        return last, had.astype(bool), li, found.astype(bool)


def update_pairs(prev_off, prev_cell, n_slots, slots, status, q_off, q_cell):
    """The pairs after an interest update, as the engine keeps them: slot slots[k] takes query k's cells (q_off / q_cell, a CSR by
    query) when status[k] == 0; a slot whose query failed, and every slot without a query, keeps its cells.  prev_off may cover fewer
    than n_slots slots (the others had none).  -> (pair_off u64[n_slots + 1], pair_cell)"""
    prev_off = np.asarray(prev_off, np.int64)
    prev_off = np.concatenate([prev_off, np.full(n_slots + 1 - len(prev_off), prev_off[-1])])
    q_off = np.asarray(q_off, np.int64)
    lens, src = np.diff(prev_off), prev_off[:-1].copy()
    ok = np.asarray(status) == 0
    s_ok = np.asarray(slots, np.int64)[ok]
    lens[s_ok] = np.diff(q_off)[ok]
    src[s_ok] = q_off[:-1][ok] + len(prev_cell)  # in the concatenation of both cell arrays
    buf = np.concatenate([np.asarray(prev_cell, np.uint32), np.asarray(q_cell, np.uint32)])
    off = np.concatenate([[0], np.cumsum(lens)])
    return off.astype(np.uint64), buf[np.repeat(src - off[:-1], lens) + np.arange(off[-1])]


def build():
    subprocess.check_call(["make", "-s", "-C", ORACLE_DIR])


def load():
    so = os.path.join(ORACLE_DIR, "libchd_oracle.so")
    src = [os.path.join(ORACLE_DIR, f) for f in ("chd_oracle.cpp", "chd_oracle.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in src):
        build()
    return Oracle(C.CDLL(so))
