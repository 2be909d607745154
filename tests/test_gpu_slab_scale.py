"""X-slab engines on one device at full scale, against the oracle: border export, halo import, re-homing, and the build, emit and
fan-out over own + halo entities.

W slab engines share one GPU and are driven through the building blocks (chd_set_slab, chd_export_border into device buffers, a
concatenation, chd_import_halo, chd_build, chd_update_interest, chd_emit_visible, chd_fanout_tick) with global ids.  Entities
move about half a cell per tick and are re-homed between ticks (the sender drops them, the receiver adopts them); subscribers
stand still on the rank that owns their centre's column.  On top of the synthetic entities sit entities on every slab boundary
(offx + k * w and its f64 neighbours), entities outside the world on each side and entities that cross a slab border every tick.
Every tick, for every subscriber of every rank:
  1. each rank's border records, the records it imports and its cell CSR equal the numpy restatements in tests/_slabs.py, and
     the CSR of every cell the rank serves holds exactly the oracle's entities of that cell, each id once;
  2. (channel, dist) pairs are bit-identical to the oracle over the whole world;
  3. the visible list is the concatenation of the rank's CSR lists of the subscriber's pairs, entry by entry (on the device), and
     on a 1 % sample it equals the oracle's visible set;
  4. chd_get_rehome lists the restated re-home set (its destinations read rank 0 on slabs without chd_comm_init, chd_gpu.h);
  5. fan-out decisions equal those of one whole-world engine for the same connections.
The capacity tests run the same checks at the border and halo capacity edges.
Run on an H100:  python -m pytest tests/test_gpu_slab_scale.py -m gpu   (about 46 s on an H100 80GB HBM3 at a 700 W limit)"""
import ctypes as C

import numpy as np
import pytest

from tests import _slabs

pytestmark = pytest.mark.gpu

MS = 1_000_000
TICK = 33 * MS
SCAN_TILE = 4096  # records per look-back tile of a compaction (chd_scan.cuh)
VIS_CHUNK = 1 << 26


@pytest.fixture(scope="module")
def chd():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from channeld_b200 import capi, engine, sharding, synth

    capi.lib()

    class NS:
        pass

    ns = NS()
    ns.torch, ns.capi, ns.engine, ns.sharding, ns.synth = torch, capi, engine, sharding, synth
    props = torch.cuda.get_device_properties(0)
    ns.l2_bytes, ns.sm_count = props.L2_cache_size, props.multi_processor_count
    return ns


class _DeviceArray:
    """A device pointer as torch sees it (__cuda_array_interface__), without a copy."""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (int(n),), "typestr": "<i4", "data": (int(ptr), False), "version": 3}


def _gather_csr(off, arr, rows):
    """The rows `rows` of a CSR (off, arr), concatenated -> (lengths, entries)"""
    off = np.asarray(off, np.int64)
    rows = np.asarray(rows, np.int64)
    lens = off[rows + 1] - off[rows]
    start = np.concatenate([[0], np.cumsum(lens)[:-1]])
    idx = np.repeat(off[rows] - start, lens) + np.arange(int(lens.sum()))
    return lens, np.asarray(arr)[idx]


def _due_set(due, conn_of_slot):
    return {(int(conn_of_slot[d["sub"]]), int(d["channel_id"]), int(d["kind"]), int(d["n_selected"]), int(d["first_sel"]), int(d["last_sel"]),
             int(d["sel_hash"]), int(d["last_message_index"]), int(d["window_hi"])) for d in due}


class _Slabs:
    """One world split into `world` X-slabs, each a slab engine on this device, plus a whole-world engine for the fan-out."""

    def __init__(self, chd, oracle, name, n_ent, n_sub, radius, world, seed=5):
        from tests._oracle import make_grid

        s = chd.synth
        self.chd, self.oracle, self.world, self.radius = chd, oracle, world, float(radius)
        wc = self.wc = s.scaled(s.CONFIGS[name], n_ent, n_sub)
        self.og = make_grid(wc.offx, wc.offz, wc.w, wc.h, wc.cols, wc.rows, wc.server_cols, wc.server_rows)
        self.halo = chd.sharding.halo_columns(radius, wc.w)
        self.slabs = [chd.sharding.slab_columns(wc.cols, world, r) for r in range(world)]
        rng = np.random.default_rng(seed)
        x, z = s.entities(wc)
        self.n_syn = n_ent
        zr = lambda n: wc.offz + rng.uniform(0.02, 0.98, n) * (wc.h * wc.rows)  # noqa: E731
        # entities on every slab boundary and one ulp to either side (three rows each)
        bx, bk = _slabs.boundary_xs(wc.offx, wc.w, wc.cols, self.slabs, self.halo)
        self.bound_x, self.bound_k = np.repeat(bx, 3), np.repeat(bk, 3)
        seeded_x = [self.bound_x]
        seeded_z = [zr(len(self.bound_x))]
        # outside the world on each side (x below, x above, z below, z above)
        x_hi, z_hi = wc.offx + wc.w * wc.cols, wc.offz + wc.h * wc.rows
        xm = wc.offx + 0.5 * wc.w
        seeded_x.append(np.array([wc.offx - 0.5 * wc.w, wc.offx - 3 * wc.w, x_hi + 0.5 * wc.w, x_hi, xm, xm, x_hi - 0.5 * wc.w, xm]))
        seeded_z.append(np.array([zr(1)[0], zr(1)[0], zr(1)[0], zr(1)[0], wc.offz - 1.0, z_hi, z_hi + 7.0, np.nextafter(wc.offz, -np.inf)]))
        # entities that cross an inner slab border every tick (a quarter cell to either side)
        inner = sorted({lo for lo, _ in self.slabs[1:]})
        self.cross_b = np.repeat(np.array(inner, np.float64), 4)
        self.n_fixed = sum(len(a) for a in seeded_x)
        self.x0 = np.concatenate([x] + seeded_x + [np.zeros(len(self.cross_b))])
        self.z0 = np.concatenate([z] + seeded_z + [zr(len(self.cross_b))])
        self.N = len(self.x0)
        self.X, self.Z = self._positions(0, self.x0[:n_ent], self.z0[:n_ent])
        # subscribers stand on synthetic entities of tick 0 and stay there, on the owner of their centre's column
        conn, cx, cz, r = s.subscribers(wc, x, z, radius)
        self.conn, self.cx, self.cz, self.r = conn, cx, cz, r
        sub_owner = chd.sharding.owner_of_column(chd.sharding.column_of(cx, wc.offx, wc.w, wc.cols), wc.cols, world)
        self.subs = [np.nonzero(sub_owner == k)[0] for k in range(world)]
        # every entity on the owner of its column; outside the world: rank 0 left of the world, the last rank right of it
        cell = self.cells()
        col = np.floor((self.X - wc.offx) / wc.w)
        own = chd.sharding.owner_of_column(np.clip(col, 0, wc.cols - 1).astype(np.int64), wc.cols, world)
        own = np.where(cell >= 0, chd.sharding.owner_of_column(cell % wc.cols, wc.cols, world), own)
        self.mine = [np.nonzero(own == k)[0] for k in range(world)]
        self.engines, self.e1 = [], None
        self.rings = None
        self.stats = dict(rehomed=0, crossings=0, seeded_exported=set(), two_away=0)

    # ---- positions
    def _positions(self, t, xs, zs):
        wc = self.wc
        side = -0.25 if t % 2 == 0 else 0.25
        xc = wc.offx + self.cross_b * wc.w + side * wc.w
        X = np.concatenate([xs, self.x0[self.n_syn:self.n_syn + self.n_fixed], xc])
        Z = np.concatenate([zs, self.z0[self.n_syn:]])
        return X, Z

    def move(self, t):
        xs, zs = self.chd.synth.move_entities(self.wc, self.X[:self.n_syn], self.Z[:self.n_syn], t, 0.5 * self.wc.w)
        prev = self.cells()
        self.X, self.Z = self._positions(t, xs, zs)
        now = self.cells()
        cols, w = self.wc.cols, self.world
        both = (prev >= 0) & (now >= 0)
        own = self.chd.sharding.owner_of_column
        self.stats["crossings"] += int((own(prev[both] % cols, cols, w) != own(now[both] % cols, cols, w)).sum())

    def cells(self):
        wc = self.wc
        return _slabs.grid_cells(self.X, self.Z, wc.offx, wc.offz, wc.w, wc.h, wc.cols, wc.rows)

    # ---- restatements of one tick
    def restate(self):
        """-> per rank dict(export, import, rehome), from the positions and the current ownership"""
        wc, cell = self.wc, self.cells()
        exports = [_slabs.export_set(cell[m], m, wc.cols, lo, hi, self.halo) for m, (lo, hi) in zip(self.mine, self.slabs)]
        out = []
        for r, (lo, hi) in enumerate(self.slabs):
            m = self.mine[r]
            out.append(dict(export=exports[r], imp=_slabs.import_set(exports, r, wc.cols, wc.cells, lo, hi, self.halo),
                            rehome=_slabs.rehome_set(cell[m], m, wc.cols, lo, hi, self.world)))
        return out

    # ---- engines
    def open(self, max_entities):
        """Slab engines of max_entities[r] entities, their lists sized from the oracle's pair and visible counts of tick 0."""
        chd, wc = self.chd, self.wc
        pw = self.oracle.sphere_pairs(self.og, self.X, self.Z, self.cx, self.cz, self.r)
        assert (pw["status"] == 0).all()
        for r, (lo, hi) in enumerate(self.slabs):
            S = len(self.subs[r])
            P = int(np.diff(pw["pair_off"].astype(np.int64))[self.subs[r]].sum())
            V = int(np.diff(pw["vis_off"].astype(np.int64))[self.subs[r]].sum())
            e = chd.engine.Engine(wc.cfg(), max_entities[r], S, max_visible=V + V // 8 + (1 << 20), max_pairs=2 * P + 4096, max_due=2 * P + 4096)
            e.set_slab(lo, hi, self.halo)
            e.set_subscribers(self.conn[self.subs[r]])
            self.engines.append(e)
        P1 = int(pw["pair_off"][-1])
        self.e1 = chd.engine.Engine(wc.cfg(), 1024, len(self.conn), max_visible=1 << 16, max_pairs=2 * P1 + 4096, max_due=2 * P1 + 4096)
        self.e1.set_subscribers(self.conn)

    def close(self):
        for e in self.engines + ([self.e1] if self.e1 is not None else []):
            e.close()
        self.engines, self.e1 = [], None

    # ---- one tick through the building blocks
    def tick(self, t, caps, parked=None, overflow_ranks=(), incomplete=()):
        """caps[r]: rank r's record capacity (its count is checked without a host read when it is short); parked[r]: extra own
        entities of rank r parked outside the world.  overflow_ranks: the ranks whose next summary must carry CHD_OVF_BORDER and
        no other bit; every other rank's must be clean.  incomplete: ranks whose halo may miss records (checked as a subset)."""
        chd, wc, torch = self.chd, self.wc, self.chd.torch
        L, t_ns = chd.capi.lib(), (t + 1) * TICK
        want = self.restate()
        cell = self.cells()
        self.rings, roff, rarr, rsnd, ridx, rcmi = chd.synth.update_rings(wc, t, t_ns, TICK, 6, len(self.conn), ring_len=32, state=self.rings)
        recs = [torch.empty(2 * max(int(c), 1), dtype=torch.int32, device="cuda") for c in caps]
        parked = parked or {}
        for r, e in enumerate(self.engines):
            m = self.mine[r]
            x, z, ids = self.X[m], self.Z[m], m.astype(np.uint32)
            k = parked.get(r, 0)
            if k:  # parked outside the world, under ids no other entity uses
                x = np.concatenate([x, np.full(k, wc.offx - 5.0 * wc.w)])
                z = np.concatenate([z, np.full(k, wc.offz + 0.5 * wc.h)])
                ids = np.concatenate([ids, np.arange(self.N, self.N + k, dtype=np.uint32)])
            e.set_entities(x, z)
            e.set_entity_ids(ids)
            e.set_rings(roff, rarr, rsnd, ridx, rcmi)
            n_exp = len(want[r]["export"][0])
            if n_exp <= caps[r]:
                assert e.export_border(recs[r], int(caps[r])) == n_exp
            else:
                e.export_border(recs[r], int(caps[r]), want_count=False)
        torch.cuda.synchronize()
        gathered = torch.cat(recs)
        torch.cuda.synchronize()
        g_host = gathered.cpu().numpy().view(np.uint32).reshape(-1, 2)
        first = np.concatenate([[0], np.cumsum(caps)]).astype(np.int64)
        n_records = int(first[-1])
        # 1a. the border records of every rank, then padding
        for r in range(self.world):
            seg = g_host[first[r]:first[r + 1]]
            gid, c = want[r]["export"]
            n = min(len(gid), int(caps[r]))
            if n == len(gid):
                np.testing.assert_array_equal(_slabs.keys(seg[:n, 0], seg[:n, 1]), _slabs.keys(gid, c), err_msg="rank %d export" % r)
            else:  # cap records of the restated set
                k = _slabs.keys(seg[:n, 0], seg[:n, 1])
                assert len(np.unique(k)) == n and np.isin(k, _slabs.keys(gid, c)).all(), r
            assert (seg[n:] == 0xFFFFFFFF).all()
            seeded = gid[(gid >= self.n_syn) & (gid < self.n_syn + self.n_fixed)]
            self.stats["seeded_exported"] |= set((cell[seeded] % wc.cols).tolist())
        # the whole world, for the oracle checks
        ocell = self.oracle.cell_of(self.og, self.X, self.Z).astype(np.int64) - self.og.channel_id_start
        ocell = np.where((ocell >= 0) & (ocell < wc.cells), ocell, -1)
        np.testing.assert_array_equal(ocell, cell)  # the restatements' cells are the oracle's
        pw = self.oracle.sphere_pairs(self.og, self.X, self.Z, self.cx, self.cz, self.r)
        self.e1.set_rings(roff, rarr, rsnd, ridx, rcmi)
        b1, k1 = chd.engine.make_batch(len(self.conn), sphere=(self.cx, self.cz, self.r))
        self.e1.update_interest(b1, t_ns)
        self.e1.fanout_tick(t_ns)
        s1 = self.e1.summary()
        assert s1.overflow == 0 and s1.n_query_errors == 0
        due1 = _due_set(self.e1.get_due(s1.n_due), self.conn)
        for r, e in enumerate(self.engines):
            lo, hi = self.slabs[r]
            subs = self.subs[r]
            e.import_halo(gathered, n_records, int(first[r]), int(caps[r]))
            e.build()
            batch, keep = chd.engine.make_batch(len(subs), sub=np.arange(len(subs), dtype=np.uint32),
                                                sphere=(self.cx[subs], self.cz[subs], self.r[subs]))
            e.update_interest(batch, t_ns)
            e.emit_visible()
            e.fanout_tick(t_ns)
            s = chd.capi.TickSummary()
            L.chd_summary(e.h, C.byref(s))
            assert s.overflow == (chd.capi.OVF_BORDER if r in overflow_ranks else 0), (r, s.overflow)
            assert s.n_query_errors == 0
            # 1b. the cell CSR: own in-world entities + the restated import, each id once
            cs, srt = e.get_cells()
            ent_cell = np.repeat(np.arange(wc.cells, dtype=np.int64), np.diff(cs.astype(np.int64)))
            assert len(np.unique(srt)) == len(srt), "rank %d: an id twice in the cell CSR" % r
            got = _slabs.keys(srt, ent_cell)
            m = self.mine[r]
            own = cell[m] >= 0
            ig, ic, isrc = want[r]["imp"]
            expect = np.sort(np.concatenate([_slabs.keys(m[own], cell[m][own]), _slabs.keys(ig, ic)]))
            if r in incomplete:  # the halo is incomplete (chd_gpu.h, CHD_OVF_BORDER): a strict subset, nothing foreign
                assert len(got) < len(expect) and np.isin(got, expect).all(), r
                continue
            np.testing.assert_array_equal(got, expect, err_msg="rank %d cell CSR" % r)
            self.stats["two_away"] += int((np.abs(isrc - r) >= 2).sum())
            a, b = _slabs.served_columns(wc.cols, lo, hi, self.halo)
            served = (ocell >= 0) & (ocell % wc.cols >= a) & (ocell % wc.cols < b)
            in_served = (ent_cell % wc.cols >= a) & (ent_cell % wc.cols < b)
            np.testing.assert_array_equal(_slabs.keys(srt[in_served], ent_cell[in_served]), _slabs.keys(np.nonzero(served)[0], ocell[served]),
                                          err_msg="rank %d served cells" % r)
            # 2. pairs, every subscriber
            p = e.get_pairs(s.n_pairs)
            plen, pch = _gather_csr(pw["pair_off"], pw["pair_cell"], subs)
            _, pdist = _gather_csr(pw["pair_off"], pw["pair_dist"], subs)
            np.testing.assert_array_equal(np.diff(p["off"].astype(np.int64)), plen)
            np.testing.assert_array_equal(p["channel"], pch)
            np.testing.assert_array_equal(p["dist"], pdist)
            # 3. visible lists: the rank's CSR lists of each subscriber's pairs, entry by entry; counts as the oracle's
            voff = np.zeros(len(subs) + 1, np.uint64)
            assert L.chd_get_visible(e.h, voff.ctypes.data_as(C.POINTER(C.c_uint64)), None) == chd.capi.OK
            np.testing.assert_array_equal(np.diff(voff.astype(np.int64)), np.diff(pw["vis_off"].astype(np.int64))[subs])
            self._check_visible(e, p, cs, srt, voff)
            sample = np.arange(0, len(subs), 100)
            j = subs[sample]
            w1 = self.oracle.sphere_tick(self.og, self.X, self.Z, self.cx[j], self.cz[j], self.r[j])
            for k, slot in enumerate(sample):
                want_vis = w1["vis_entity"][int(w1["vis_off"][k]):int(w1["vis_off"][k + 1])]
                np.testing.assert_array_equal(np.sort(e.get_visible_slot(int(slot), cap=1 << 22)), np.sort(want_vis))
            # 5. fan-out decisions
            conn_of_slot = self.conn[subs]
            mine_conn = set(conn_of_slot.tolist())
            assert _due_set(e.get_due(s.n_due), conn_of_slot) == {d for d in due1 if d[0] in mine_conn}, "rank %d due" % r
        del gathered
        # 4. re-homing: sender drops, receiver adopts
        moves = []
        for r, e in enumerate(self.engines):
            gid, dst, n = e.get_rehome(cap=1 << 22)
            wg, wd = want[r]["rehome"]
            assert n == len(wg)
            np.testing.assert_array_equal(np.sort(gid.astype(np.int64)), np.sort(wg), err_msg="rank %d rehome" % r)
            # a slab made with chd_set_slab alone knows no world: it names rank 0 as every destination (chd_gpu.h), and the host
            # that chose the slabs routes by column
            assert (dst == 0).all()
            moves.append((wg, wd))
        self.stats["rehomed"] += sum(len(g) for g, _ in moves)
        for r in range(self.world):
            adopt = np.concatenate([g[d == r] for g, d in moves])
            self.mine[r] = np.union1d(np.setdiff1d(self.mine[r], moves[r][0]), adopt)
        return want, n_records

    def _check_visible(self, e, p, cs, srt, voff):
        """vis_entity[voff[s] ..] = the CSR lists of slot s's pair cells, in pair order; compared on the device in chunks"""
        torch, chd = self.chd.torch, self.chd
        V = int(voff[-1])
        ptr, n = e.device_view(chd.capi.VIEW_VIS_ENTITY)
        assert n >= V
        vis = torch.as_tensor(_DeviceArray(ptr, n), device="cuda")[:V]
        cell = p["channel"].astype(np.int64) - self.og.channel_id_start
        cs64 = cs.astype(np.int64)
        length = cs64[cell + 1] - cs64[cell]
        cum = np.concatenate([[0], np.cumsum(length)])
        np.testing.assert_array_equal(cum[p["off"].astype(np.int64)], voff.astype(np.int64))
        srt_t = torch.from_numpy(srt.view(np.int32)).cuda()
        delta_t = torch.from_numpy(cs64[cell] - cum[:-1]).cuda()
        len_t = torch.from_numpy(length).cuda()
        P = len(cell)
        i = 0
        while i < P:
            j = min(P, max(i + 1, int(np.searchsorted(cum, cum[i] + VIS_CHUNK, "right")) - 1))
            a, b = int(cum[i]), int(cum[j])
            if b > a:
                idx = torch.repeat_interleave(delta_t[i:j], len_t[i:j], output_size=b - a) + torch.arange(a, b, device="cuda")
                same = srt_t[idx] == vis[a:b]
                if not bool(same.all()):
                    k = a + int(torch.nonzero(~same)[0, 0])
                    pytest.fail("visible entry %d: %d, CSR says %d" % (k, int(vis[k]), int(srt_t[idx[k - a]])))
            i = j
        torch.cuda.synchronize()


def _caps_with_margin(want, floor=0):
    return [max(len(w["export"][0]) + len(w["export"][0]) // 5 + 1024, floor) for w in want]


def _max_entities(sl, want, caps, extra=0):
    n_records = sum(caps)
    return [max(n_records, len(sl.mine[r]) + len(want[r]["imp"][0])) + extra for r in range(sl.world)]


# name, entities, subscribers, radius, slabs, ticks, emit kernel side, import compaction beyond the SM count
RUNS = {
    "benchmark-w2": ("benchmark", 1_000_000, 20_000, 50.0, 2, 3, "cta", True),
    "benchmark-w8": ("benchmark", 1_000_000, 20_000, 2500.0, 8, 3, "cta", False),
    "2x2-w2": ("2x2", 50_000, 2_000, 500.0, 2, 4, "cta", False),
    "handover-w3": ("handover", 200_000, 4_000, 50.0, 3, 4, "warp", False),
}


@pytest.mark.parametrize("run", list(RUNS))
def test_slabs_at_scale(chd, oracle, run):
    name, n_ent, n_sub, radius, world, n_ticks, side, wide_import = RUNS[run]
    sl = _Slabs(chd, oracle, name, n_ent, n_sub, radius, world)
    try:
        wc = sl.wc
        want = sl.restate()
        caps = _caps_with_margin(want)
        if wide_import:  # a halo import whose compaction spans more look-back tiles than the device has SMs
            caps = _caps_with_margin(want, (chd.sm_count + 1) * SCAN_TILE // world + 1)
            assert -(-sum(caps) // SCAN_TILE) > chd.sm_count
        widths = [hi - lo for lo, hi in sl.slabs]
        if run == "benchmark-w8":
            assert sl.halo == 2 and min(widths) < sl.halo  # a halo wider than a slab: records come from two ranks away
        if name == "2x2":
            assert widths == [1, 1] and sl.halo == 1  # one-column slabs, no interior
        # the emit kernel each slab takes (chd_tick.cu emit_uses_cta_tiles; no chd_comm_init: border capacity 0)
        for r, (lo, hi) in enumerate(sl.slabs):
            n_own = len(sl.mine[r])
            assert _slabs.emit_uses_cta_tiles(n_own, hi - lo, wc.rows, n_own, chd.l2_bytes) == (side == "cta"), (r, n_own)
        sl.open([m + m // 8 + 4096 for m in _max_entities(sl, want, caps)])
        for t in range(n_ticks):
            if t:
                sl.move(t)
            w = sl.restate()
            assert all(len(w[r]["export"][0]) <= caps[r] for r in range(world))
            sl.tick(t, caps)
        st = sl.stats
        # every column the seeded boundary entities fall in that another rank serves was exported with them
        bcell = sl.cells()[sl.n_syn:sl.n_syn + len(sl.bound_x)]
        need = {c for c in set((bcell[bcell >= 0] % wc.cols).tolist()) if _needed_elsewhere(sl, c)}
        assert need and need <= st["seeded_exported"], (need - st["seeded_exported"])
        assert st["rehomed"] > 0 and st["crossings"] > 0, st
        if run == "benchmark-w8":
            assert st["two_away"] > 0
    finally:
        sl.close()


def _needed_elsewhere(sl, col):
    """some rank other than the column's owner serves it"""
    owner = int(sl.chd.sharding.owner_of_column(col, sl.wc.cols, sl.world))
    return any(r != owner and _slabs.served_columns(sl.wc.cols, lo, hi, sl.halo)[0] <= col < _slabs.served_columns(sl.wc.cols, lo, hi, sl.halo)[1]
               for r, (lo, hi) in enumerate(sl.slabs))


CAP_WORLD = ("benchmark", 1_000_000, 5_000, 50.0, 2)


def test_border_capacity_edge(chd, oracle):
    """cap = the restated border count: no overflow, exact.  cap - 1 on rank 0: CHD_OVF_BORDER in rank 0's next summary, and rank 1's
    halo is incomplete.  Then cap again: exact."""
    sl = _Slabs(chd, oracle, *CAP_WORLD)
    try:
        want = sl.restate()
        exact = [len(w["export"][0]) for w in want]
        sl.open(_max_entities(sl, want, exact, 4096))
        sl.tick(0, exact)
        sl.tick(1, [exact[0] - 1, exact[1]], overflow_ranks=(0,), incomplete=(1,))
        sl.tick(2, exact)
    finally:
        sl.close()


def test_halo_capacity_edge(chd, oracle):
    """max_entities = own + halo exactly: no overflow, exact.  One own entity more (parked outside the world) on rank 0: the build
    length is clamped, CHD_OVF_BORDER in rank 0's next summary and its halo is incomplete.  Then back to own + halo: exact."""
    sl = _Slabs(chd, oracle, *CAP_WORLD)
    try:
        want = sl.restate()
        caps = [len(w["export"][0]) for w in want]
        sl.open([len(sl.mine[r]) + len(want[r]["imp"][0]) for r in range(sl.world)])
        assert all(sum(caps) <= len(sl.mine[r]) + len(want[r]["imp"][0]) for r in range(sl.world))
        sl.tick(0, caps)
        sl.tick(1, caps, parked={0: 1}, overflow_ranks=(0,), incomplete=(0,))
        sl.tick(2, caps)
    finally:
        sl.close()
