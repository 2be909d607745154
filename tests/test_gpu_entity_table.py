"""Entity-table mode (chd_entity_table_init): entities spawned, moved and despawned by id, every result reported in ids.  A Python
model of the table (the documented slot policy, statuses and counters) plus the oracle's cell_of / sphere_tick give the expected
cells, visible lists, pairs, handovers and visible-set deltas.
Run on an H100:  python -m pytest tests -m gpu"""
import ctypes as C
import os
from collections import deque

import numpy as np
import pytest

from tests.test_gpu_visible_delta import _set_diff

gpu = pytest.mark.gpu
MS = 1_000_000
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_entity_stats_layout_matches_header(tmp_path):
    """chd_entity_stats compiles as C99 and the ctypes mirror has the C compiler's size and field offsets (no GPU needed)."""
    import subprocess

    from channeld_b200 import capi

    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "chd_gpu.h"', 'int main(void) {',
             '  printf("size %zu\\n", sizeof(chd_entity_stats));']
    lines += ['  printf("%s %%zu\\n", offsetof(chd_entity_stats, %s));' % (f, f) for f, _ in capi.EntityStats._fields_]
    lines += ['  return CHD_EV_OK + CHD_EV_DUPLICATE + CHD_EV_UNKNOWN_ID + CHD_EV_RESERVED_ID + CHD_EV_TABLE_FULL - 10 + CHD_VIEW_ENTITY_ID - 13;', '}']
    src = tmp_path / "stats.c"
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "stats"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())
    assert int(got["size"]) == C.sizeof(capi.EntityStats) == 4 * 4 + 4 * 8
    for f, _ in capi.EntityStats._fields_:
        assert int(got[f]) == getattr(capi.EntityStats, f).offset, f
    assert (capi.EV_OK, capi.EV_DUPLICATE, capi.EV_UNKNOWN_ID, capi.EV_RESERVED_ID, capi.EV_TABLE_FULL) == (0, 1, 2, 3, 4)


@pytest.fixture(scope="module")
def chd():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from channeld_b200 import capi, controller, engine, synth

    capi.lib()

    class NS:
        pass

    ns = NS()
    ns.capi, ns.controller, ns.engine, ns.synth = capi, controller, engine, synth
    return ns


RESERVED = (0, 0xFFFFFFFF)


class Model:
    """The table as chd_gpu.h specifies it: released slots first in first out, then fresh ones; with deltas on, a despawned slot is
    held until the summary of the tick that built without it (every tick here reads its summary and its delta succeeds)."""

    def __init__(self, n_max, deltas):
        self.N, self.deltas = n_max, deltas
        self.slot_of = {}
        self.id_of = np.zeros(n_max, np.uint32)
        self.inst_of = np.zeros(n_max, np.int64)  # instance number of the entity in each slot (a respawn is a new instance)
        self.inst_id = [0]
        self.x = np.full(n_max, np.nan)
        self.z = np.full(n_max, np.nan)
        self.fifo, self.held, self.hw = deque(), [], 0
        self.flagged = set()  # slots spawned / despawned since the last build
        self.applied = self.unknown = self.superseded = 0
        self.prev = None  # (id_of, cell) per slot at the last build

    def spawn(self, ids, x, z, f32):
        if f32:
            x, z = np.float32(x).astype(np.float64), np.float32(z).astype(np.float64)
        st, seen = [], set()
        for i, id_ in enumerate(int(v) for v in ids):
            if id_ in RESERVED:
                st.append(3)
                continue
            dup = id_ in seen or id_ in self.slot_of
            seen.add(id_)
            if dup:
                st.append(1)
                continue
            if self.fifo:
                slot = self.fifo.popleft()
            elif self.hw < self.N:
                slot, self.hw = self.hw, self.hw + 1
            else:
                st.append(4)
                continue
            self.slot_of[id_] = slot
            self.id_of[slot], self.x[slot], self.z[slot] = id_, x[i], z[i]
            self.inst_of[slot] = len(self.inst_id)
            self.inst_id.append(id_)
            self.flagged.add(slot)
            st.append(0)
        return np.array(st, np.uint8)

    def despawn(self, ids):
        st, seen = [], set()
        for id_ in (int(v) for v in ids):
            if id_ in RESERVED:
                st.append(3)
                continue
            if id_ in seen:
                st.append(1)
                continue
            seen.add(id_)
            if id_ not in self.slot_of:
                st.append(2)
                continue
            slot = self.slot_of.pop(id_)
            self.id_of[slot], self.inst_of[slot], self.x[slot], self.z[slot] = 0, 0, np.nan, np.nan
            self.flagged.add(slot)
            (self.held if self.deltas else self.fifo).append(slot)
            st.append(0)
        return np.array(st, np.uint8)

    def move(self, ids, x, z, f32):
        if f32:
            x, z = np.float32(x).astype(np.float64), np.float32(z).astype(np.float64)
        last = {}
        for i, id_ in enumerate(int(v) for v in ids):
            if id_ in self.slot_of:
                last[id_] = i
            else:
                self.unknown += 1
        live = sum(1 for v in ids if int(v) in self.slot_of)
        for id_, i in last.items():
            s = self.slot_of[id_]
            self.x[s], self.z[s] = x[i], z[i]
        self.applied += len(last)
        self.superseded += live - len(last)

    def after_summary(self):
        self.fifo.extend(self.held)
        self.held = []


class World:
    def __init__(self, chd, oracle, name, n0, n_max, n_sub, radius, seed):
        self.wc = chd.synth.CONFIGS[name]
        g = self.wc
        from tests._oracle import make_grid

        self.og = make_grid(g.offx, g.offz, g.w, g.h, g.cols, g.rows, g.server_cols, g.server_rows)
        self.lo_x, self.lo_z = g.offx, g.offz
        self.hi_x, self.hi_z = g.offx + g.w * g.cols, g.offz + g.h * g.rows
        self.far = self.hi_x + 50 * g.w  # outside the world (the oracle's stand-in for a parked slot)
        self.n0, self.N, self.S = n0, n_max, n_sub
        rng = np.random.default_rng(seed + 1000)
        self.cx = rng.uniform(self.lo_x + 1, self.hi_x - 1, n_sub)
        self.cz = rng.uniform(self.lo_z + 1, self.hi_z - 1, n_sub)
        self.r = rng.uniform(radius[0], radius[1], n_sub)
        self.oracle = oracle

    def pos(self, rng, k, out_frac=0.03):
        x = rng.uniform(self.lo_x, self.hi_x, k)
        z = rng.uniform(self.lo_z, self.hi_z, k)
        out = rng.random(k) < out_frac
        x[out] = self.far
        return x, z

    def cells(self, m):
        x = np.where(np.isnan(m.x[:m.hw]), self.far, m.x[:m.hw])
        z = np.where(np.isnan(m.z[:m.hw]), self.far, m.z[:m.hw])
        return x, z, self.oracle.cell_of(self.og, x, z)


def tick_ops(rng, w, m, t, state):
    """The events of tick t: despawns (with an unknown and a reserved id and a repeat), spawns (same-tick and next-tick respawns,
    fresh ids that grow the high-water mark, a repeat, a live id, a reserved id; f32 on odd ticks), moves (in-call duplicates,
    unknown ids, entities leaving and re-entering the world; f32 every third tick)."""
    if t == 0:
        ids = rng.permutation(np.unique(rng.integers(7, 1 << 31, w.n0 + w.n0 // 8)))[:w.n0].astype(np.uint32)  # sparse 31-bit ids
        state["next"] = int(ids.max()) + 1
        x, z = w.pos(rng, w.n0)
        return [("spawn", ids, x, z, False)]
    live = np.array(sorted(m.slot_of), np.uint32)
    k = max(4, len(live) // 400)
    dead = rng.choice(live, k, replace=False)
    ops = [("despawn", np.concatenate([dead, np.array([state["next"] + 12345, 0, dead[0]], np.uint32)]))]
    fresh = np.arange(state["next"], state["next"] + k + max(2, k // 4), dtype=np.uint32)
    state["next"] += len(fresh)
    sp = np.concatenate([dead[:k // 3], state.get("dead", dead)[k // 3:2 * k // 3], fresh, fresh[:1], np.array([0xFFFFFFFF], np.uint32), live[-1:]])
    state["dead"] = dead
    x, z = w.pos(rng, len(sp))
    ops.append(("spawn", sp, x, z, t % 2 == 1))
    mv = rng.choice(live, max(8, len(live) // 10), replace=False)
    mv = np.concatenate([mv, mv[:len(mv) // 20], dead[2 * k // 3:], np.array([0], np.uint32)])
    x, z = w.pos(rng, len(mv), out_frac=0.05)
    ops.append(("move", mv.astype(np.uint32), x, z, t % 3 == 0))
    return ops


def apply(chd, e, m, op):
    kind = op[0]
    if kind == "spawn":
        _, ids, x, z, f32 = op
        got = (e.spawn_entities_f32 if f32 else e.spawn_entities)(ids, x, z)
        want = m.spawn(ids, x, z, f32)
    elif kind == "despawn":
        got = e.despawn_entities(op[1])
        want = m.despawn(op[1])
    else:
        _, ids, x, z, f32 = op
        (e.move_entities_f32 if f32 else e.move_entities)(ids, x, z)
        m.move(ids, x, z, f32)
        return
    np.testing.assert_array_equal(got, want, err_msg=kind)


def table_engine(chd, w, graphs=True):
    e = chd.engine.Engine(w.wc.cfg(), w.N, w.S)
    e.enable_graphs(graphs)
    e.entity_table_init()
    e.set_subscribers(np.arange(1, w.S + 1, dtype=np.uint32))
    e.reserve_visible_delta(1 << 22)
    return e


def batch(chd, w, t):
    """-> (query batch, radii): some subscriptions change every tick"""
    r = w.r * (1.0 + 0.25 * ((np.arange(w.S) + t) % 3))
    b, keep = chd.engine.make_batch(w.S, sub=np.arange(w.S, dtype=np.uint32), sphere=(w.cx, w.cz, r))
    b._keep = keep
    return b, r


@gpu
@pytest.mark.parametrize("name,n0,n_max,n_sub,radius", [("2x2", 900, 1400, 64, (50.0, 2500.0)),
                                                       ("benchmark", 232_000, 250_000, 300, (30.0, 120.0))])
def test_model_run(chd, oracle, name, n0, n_max, n_sub, radius):
    """12 ticks of random events, each tick chd_tick(TICK_ALL | TICK_VISIBLE_DELTA), checked in ids against the model and the oracle:
    every cell's entities (slot order), the visible lists (also = the concatenation of their pairs' CSR lists), the pairs, the
    handover set and the delta as instance-set differences.  The two worlds sit on either side of the emit kernel choice."""
    w = World(chd, oracle, name, n0, n_max, n_sub, radius, seed=7)
    e = table_engine(chd, w)
    m = Model(w.N, deltas=True)
    rng = np.random.default_rng(7)
    state, prev_vis = {}, (np.zeros(w.S + 1, np.uint64), np.zeros(0, np.int64))
    id_start = w.wc.cfg().channel_id_start
    handovers = 0
    for t in range(12):
        for op in tick_ops(rng, w, m, t, state):
            apply(chd, e, m, op)
        b, r = batch(chd, w, t)
        s = e.tick(b, (t + 1) * 33 * MS, chd.capi.TICK_ALL | chd.capi.TICK_VISIBLE_DELTA)
        x, z, cell = w.cells(m)
        # cell CSR: in-world slots by (cell, slot), named by id
        inw = np.nonzero(cell)[0]
        order = inw[np.lexsort((inw, cell[inw]))]
        cs_want = np.concatenate([[0], np.cumsum(np.bincount(cell[inw] - id_start, minlength=w.og.grid_cols * w.og.grid_rows))]).astype(np.uint32)
        cs, se = e.get_cells()
        np.testing.assert_array_equal(cs, cs_want)
        np.testing.assert_array_equal(se, m.id_of[order])
        assert s.n_entities_in_world == len(inw)
        # pairs and visible lists
        want = oracle.sphere_tick(w.og, x, z, w.cx, w.cz, r)
        pairs = e.get_pairs()
        np.testing.assert_array_equal(pairs["off"], want["pair_off"])
        np.testing.assert_array_equal(pairs["channel"], want["pair_cell"])
        voff, vis = e.get_visible()
        np.testing.assert_array_equal(voff, want["vis_off"])
        np.testing.assert_array_equal(vis, m.id_of[want["vis_entity"]])
        po = pairs["off"]
        for sub in range(0, w.S, max(1, w.S // 40)):
            cat = [se[cs[c - id_start]:cs[c - id_start + 1]] for c in pairs["channel"][po[sub]:po[sub + 1]]]
            np.testing.assert_array_equal(vis[voff[sub]:voff[sub + 1]], np.concatenate(cat) if cat else np.zeros(0, np.uint32))
        # handovers: live at both builds, same instance, not spawned / despawned in between, cell changed
        ho = e.get_handover(s.n_handover)
        got = set(zip(*(a.tolist() for a in ho)))
        assert len(got) == s.n_handover
        want_ho = set()
        if m.prev is not None:
            pid, pcell = m.prev
            k = min(len(pid), m.hw)
            sl = np.arange(k)
            keep_ = (m.id_of[:k] != 0) & (pid[:k] == m.id_of[:k]) & (pcell[:k] != cell[:k]) & ~np.isin(sl, list(m.flagged))
            want_ho = set(zip(m.id_of[:k][keep_].tolist(), pcell[:k][keep_].tolist(), cell[:k][keep_].tolist()))
        assert got == want_ho, t
        handovers += len(got)
        m.prev, m.flagged = (m.id_of[:m.hw].copy(), cell.copy()), set()
        # visible-set delta: instance-set differences, reported by id in the engine's order
        now_vis = (want["vis_off"], m.inst_of[want["vis_entity"]])
        eo, en, lo, le = _set_diff(prev_vis, now_vis, w.S)
        inst_id = np.array(m.inst_id, np.uint32)
        got_d = e.get_visible_delta()
        np.testing.assert_array_equal(got_d[0], eo)
        np.testing.assert_array_equal(got_d[1], inst_id[en])
        np.testing.assert_array_equal(got_d[2], lo)
        np.testing.assert_array_equal(got_d[3], inst_id[le])
        prev_vis = now_vis
        m.after_summary()
        st = e.entity_stats()
        assert (st["live"], st["high_water"], st["quarantined"]) == (len(m.slot_of), m.hw, 0)
        assert st["free_slots"] == len(m.fifo) + m.N - m.hw
        assert (st["moves_applied"], st["moves_unknown"], st["moves_superseded"]) == (m.applied, m.unknown, m.superseded)
    assert handovers > 0 and m.hw > n0


@gpu
def test_quarantine_survives_a_delta_overflow(chd):
    """A slot despawned while deltas are on stays quarantined through CHD_OVF_DELTA ticks; after a re-reserve the next delta reports
    the old instance in leave and the new one (same id, fresh slot) in enter, and only then is the slot released."""
    cap = chd.capi
    L = cap.lib()
    wc = chd.synth.CONFIGS["2x2"]
    e = chd.engine.Engine(wc.cfg(), 64, 2)
    e.entity_table_init()
    e.set_subscribers(np.array([1, 2], np.uint32))
    e.reserve_visible_delta(16)
    b, keep = chd.engine.make_batch(1, sub=np.array([0], np.uint32), sphere=(np.array([0.0]), np.array([0.0]), np.array([5000.0])))

    def tick():
        s = cap.TickSummary()
        st = L.chd_tick(e.h, C.byref(b), 0, cap.TICK_ALL | cap.TICK_VISIBLE_DELTA, C.byref(s))
        return st, s

    xy = lambda ids: (np.asarray(ids, np.float64) * 10.0 - 300.0, np.asarray(ids, np.float64) * 7.0 - 200.0)
    ids = np.arange(1, 9, dtype=np.uint32)
    assert (e.spawn_entities(ids, *xy(ids)) == 0).all()
    assert tick()[0] == cap.OK
    assert sorted(e.get_visible_delta()[1].tolist()) == list(range(1, 9))
    assert (e.despawn_entities([3]) == 0).all()
    more = np.arange(9, 41, dtype=np.uint32)
    assert (e.spawn_entities(more, *xy(more)) == 0).all()  # 32 entries to enter: more than 16
    st, s = tick()
    assert st == cap.ERR_CAPACITY and s.overflow == cap.OVF_DELTA
    assert e.entity_stats()["quarantined"] == 1
    assert (e.spawn_entities([3], *xy([3])) == 0).all()  # a new instance of id 3: a fresh slot, slot 2 is held
    st, s = tick()
    assert st == cap.ERR_CAPACITY and e.entity_stats()["quarantined"] == 1 and e.entity_stats()["high_water"] == 41
    e.reserve_visible_delta(4096)
    st, s = tick()
    assert st == cap.OK
    eo, en, lo, le = e.get_visible_delta()
    assert le.tolist() == [3]
    assert sorted(en.tolist()) == list(range(3, 4)) + list(range(9, 41))
    stats = e.entity_stats()
    assert stats["quarantined"] == 0 and stats["free_slots"] == 1 + 64 - 41 and stats["live"] == 40
    assert (e.spawn_entities([100], *xy([100])) == 0).all()  # takes the released slot: the high-water mark stays
    assert e.entity_stats()["high_water"] == 41


@gpu
def test_statuses_and_counters(chd):
    """Every rejection status, with the table untouched by rejected events; move counters (last move of an id in a call wins)."""
    cap = chd.capi
    wc = chd.synth.CONFIGS["2x2"]
    e = chd.engine.Engine(wc.cfg(), 8, 1)
    e.entity_table_init()
    E = cap
    pos = lambda k: (np.linspace(-1500, 1500, k), np.linspace(-1000, 1000, k))
    assert e.spawn_entities([5, 0, 5, 0xFFFFFFFF, 6], *pos(5)).tolist() == [E.EV_OK, E.EV_RESERVED_ID, E.EV_DUPLICATE, E.EV_RESERVED_ID, E.EV_OK]
    assert e.spawn_entities([5], *pos(1)).tolist() == [E.EV_DUPLICATE]
    assert e.despawn_entities([7, 0, 6, 6, 0xFFFFFFFF]).tolist() == [E.EV_UNKNOWN_ID, E.EV_RESERVED_ID, E.EV_OK, E.EV_DUPLICATE, E.EV_RESERVED_ID]
    ids = np.arange(10, 21, dtype=np.uint32)
    st = e.spawn_entities(ids, *pos(11))
    assert st.tolist() == [E.EV_OK] * 7 + [E.EV_TABLE_FULL] * 4
    s = e.entity_stats()
    assert (s["live"], s["high_water"], s["free_slots"], s["quarantined"]) == (8, 8, 0, 0)
    e.build()
    cs, se = e.get_cells()
    assert sorted(se.tolist()) == [5] + list(range(10, 17))
    # moves: 5 twice (the second wins), 99 and 0 unknown, 10 once
    e.move_entities([5, 5, 99, 10, 0], [1900.0, -1900.0, 0.0, 1900.0, 0.0], [1900.0, -1900.0, 0.0, 1900.0, 0.0])
    s = e.entity_stats()
    assert (s["moves_applied"], s["moves_unknown"], s["moves_superseded"]) == (2, 2, 1)
    e.build()
    cs, se = e.get_cells()
    cell_of = {int(v): c for c in range(4) for v in se[cs[c]:cs[c + 1]]}
    assert cell_of[5] == 0 and cell_of[10] == 3  # (-1900, -1900): cell 0; (1900, 1900): the last cell of the 2x2 grid
    # despawned ids vanish, a failed despawn changes nothing
    assert e.despawn_entities([5, 5]).tolist() == [E.EV_OK, E.EV_DUPLICATE]
    e.build()
    assert sorted(e.get_cells()[1].tolist()) == list(range(10, 17))
    c = chd.controller.GpuStaticGrid2DSpatialController(max_entities=16, max_subscribers=4)
    c.LoadConfig({"GridWidth": 2000, "GridHeight": 2000, "GridCols": 2, "GridRows": 2, "ServerCols": 1, "ServerRows": 2,
                  "WorldOffsetX": -2000, "WorldOffsetZ": -2000})
    assert c.SpawnObjects([42, 43], [-100.0, 100.0], [-100.0, 100.0]).tolist() == [0, 0]
    c.MoveEntities([43], [-100.0], [-100.0])
    assert c.DestroyObjects([42, 44]).tolist() == [E.EV_OK, E.EV_UNKNOWN_ID]
    c.engine.build()
    assert c.engine.get_cells()[1].tolist() == [43]


def _run_arrays(chd, oracle, w, graphs, ticks=8):
    e = table_engine(chd, w, graphs)
    m = Model(w.N, deltas=True)
    rng = np.random.default_rng(11)
    state, out = {}, []
    for t in range(ticks):
        for op in tick_ops(rng, w, m, t, state):
            apply(chd, e, m, op)
        b, keep = batch(chd, w, t)
        s = e.tick(b, (t + 1) * 33 * MS, chd.capi.TICK_ALL | chd.capi.TICK_VISIBLE_DELTA)
        m.after_summary()
        ho = e.get_handover(s.n_handover)
        out.append([*e.get_cells(), *e.get_visible(), *e.get_visible_delta(), np.sort((ho[0].astype(np.uint64) << np.uint64(32)) | ho[1])])
    return out, e.graph_launch_count()


@gpu
def test_deterministic_with_and_without_graphs(chd, oracle):
    """The same event sequence on two engines, CUDA graphs on and off: identical cell CSRs, visible lists, deltas and handovers."""
    w = World(chd, oracle, "2x2", 900, 1400, 64, (50.0, 2500.0), seed=3)
    a, ga = _run_arrays(chd, oracle, w, True)
    b, gb = _run_arrays(chd, oracle, w, False)
    assert ga > 0 and gb == 0
    for t, (ra, rb) in enumerate(zip(a, b)):
        for k, (u, v) in enumerate(zip(ra, rb)):
            np.testing.assert_array_equal(u, v, err_msg="tick %d array %d" % (t, k))


@gpu
def test_async_read_back_reports_ids(chd, oracle):
    """chd_fetch_results_async / chd_fetch_wait return the id-valued cell CSR and handover list, equal to a synchronous fetch."""
    import torch

    cap = chd.capi
    L = cap.lib()
    w = World(chd, oracle, "2x2", 900, 1400, 64, (50.0, 2500.0), seed=5)
    e = table_engine(chd, w)
    m = Model(w.N, deltas=True)
    rng = np.random.default_rng(5)
    state = {}
    C1 = w.og.grid_cols * w.og.grid_rows + 1
    pin = lambda k: torch.zeros(k, dtype=torch.int32).pin_memory()
    cs_t, se_t, he_t, hs_t, hd_t, hdr_t = pin(C1), pin(w.N), pin(w.N), pin(w.N), pin(w.N), pin(64)
    rb = cap.ResultBuffers()
    rb.cell_start, rb.sorted_entity, rb.entity_cap = cap.ptr(cs_t), cap.ptr(se_t), w.N
    rb.handover_entity, rb.handover_src, rb.handover_dst, rb.handover_cap = cap.ptr(he_t), cap.ptr(hs_t), cap.ptr(hd_t), w.N
    cs_n, se_n, he_n, hs_n, hd_n = np.zeros(C1, np.uint32), *(np.zeros(w.N, np.uint32) for _ in range(4))
    rs = cap.ResultBuffers()
    rs.cell_start, rs.sorted_entity, rs.entity_cap = cap.ptr(cs_n), cap.ptr(se_n), w.N
    rs.handover_entity, rs.handover_src, rs.handover_dst, rs.handover_cap = cap.ptr(he_n), cap.ptr(hs_n), cap.ptr(hd_n), w.N
    seen_ho = 0
    for t in range(4):
        for op in tick_ops(rng, w, m, t, state):
            apply(chd, e, m, op)
        b, keep = batch(chd, w, t)
        e.tick(b, (t + 1) * 33 * MS, cap.TICK_ALL | cap.TICK_EARLY_RESULTS | cap.TICK_VISIBLE_DELTA, want_summary=False)
        s = cap.TickSummary()
        assert L.chd_fetch_results_async(e.h, C.byref(rb), cap.ptr(hdr_t)) == cap.OK
        assert L.chd_fetch_wait(e.h, C.byref(s)) == cap.OK
        m.after_summary()
        s2 = cap.TickSummary()
        assert L.chd_fetch_results(e.h, C.byref(rs), C.byref(s2)) == cap.OK
        nin, nh = s.n_entities_in_world, s.n_handover
        assert (nin, nh) == (s2.n_entities_in_world, s2.n_handover)
        np.testing.assert_array_equal(cs_t.numpy().view(np.uint32), cs_n)
        np.testing.assert_array_equal(se_t.numpy().view(np.uint32)[:nin], se_n[:nin])
        cs, se = e.get_cells()
        np.testing.assert_array_equal(se, se_n[:nin])
        assert set(se.tolist()) <= set(m.slot_of)
        trip = lambda a, b_, c: set(zip(a[:nh].tolist(), b_[:nh].tolist(), c[:nh].tolist()))
        got = trip(he_t.numpy().view(np.uint32), hs_t.numpy().view(np.uint32), hd_t.numpy().view(np.uint32))
        assert got == trip(he_n, hs_n, hd_n) == trip(*e.get_handover(nh))
        assert {h[0] for h in got} <= set(m.slot_of)
        seen_ho += nh
    assert seen_ho > 0


@gpu
def test_long_churn_rebuilds_the_device_table(chd, oracle):
    """Despawns leave tombstones until live entries + tombstones pass 3/4 of the table and it is rebuilt from the host map; moves
    keep resolving through every rebuild."""
    w = World(chd, oracle, "2x2", 200, 256, 4, (50.0, 100.0), seed=9)
    e = chd.engine.Engine(w.wc.cfg(), w.N, w.S)
    e.entity_table_init()
    m = Model(w.N, deltas=False)
    rng = np.random.default_rng(9)
    ids = np.arange(1000, 1200, dtype=np.uint32)
    apply(chd, e, m, ("spawn", ids, *w.pos(rng, 200, 0.0), False))
    nxt = 1200
    for r in range(12):
        live = np.array(sorted(m.slot_of), np.uint32)
        dead = rng.choice(live, 40, replace=False)
        apply(chd, e, m, ("despawn", dead))
        fresh = np.arange(nxt, nxt + 40, dtype=np.uint32)
        nxt += 40
        apply(chd, e, m, ("spawn", fresh, *w.pos(rng, 40, 0.0), r % 2 == 1))
        live = np.array(sorted(m.slot_of), np.uint32)
        apply(chd, e, m, ("move", live, *w.pos(rng, len(live), 0.1), r % 2 == 0))
        e.build()
        x, z, cell = w.cells(m)
        inw = np.nonzero(cell)[0]
        order = inw[np.lexsort((inw, cell[inw]))]
        np.testing.assert_array_equal(e.get_cells()[1], m.id_of[order])
    s = e.entity_stats()
    assert s["rebuilds"] >= 2
    assert (s["moves_applied"], s["moves_unknown"], s["moves_superseded"]) == (m.applied, 0, 0)
    assert s["live"] == 200 and s["high_water"] == 200  # (no deltas: every despawned slot is reused by the next spawn call)
