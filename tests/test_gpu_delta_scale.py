"""Visible-set deltas (CHD_TICK_VISIBLE_DELTA) against the oracle's set-difference delta (orc_visible_delta) at the sizes where the
delta kernels loop: every grid-stride loop of the stage runs more than once, and the slot-offset scans run over more than 32 tiles.

Constants the sizes depend on (SM count from torch):
  DELTA_THREADS = 256                chd_delta.cuh: block size of every delta kernel
  TBL_THREADS = 256                  chd_table.cuh: block size of the table's delta kernels
  SCAN_TILE = 4096                   chd_scan.cuh: SCAN_THREADS x SCAN_ITEMS entries per look-back tile
  LOOKBACK_HOP = 32                  chd_scan.cuh: predecessor descriptors one look-back hop reads
  delta_slots_kernel                 chd_delta.cu: at most 32 x SMs blocks, one warp per slot -> loops past 256 x SMs slots
  delta_moves_kernel, delta_advance_kernel, delta_id_scatter_kernel
                                     chd_delta.cu: 8 x SMs blocks -> loop past 2048 x SMs entities, pairs or cells
  tbl_delta_ids_kernel, tbl_delta_commit_kernel
                                     chd_table.cu: 8 x SMs blocks of TBL_THREADS -> loop past 2048 x SMs entries or entities

  case  mode          world                                             loops it is sized to take twice
  A     index         100 x 100 cells, 400 K entities, 160 K slots      slots, moves (entities), advance (entities, pairs)
  B     index         600 x 600 cells, 500 K entities, 50 K slots       moves' per-cell starts (cells + 1), advance (cells + 2)
  C     index         the benchmark world beside emit and fan-out       slots, moves, advance
  D     id            case A's world, ids in [0, 2^21), array permuted  A's loops and the id scatter
  E     entity table  400 K spawned ids, 160 K slots                    A's loops, the table's id translation and commit
Run on an H100:  python -m pytest tests/test_gpu_delta_scale.py -m gpu
"""
import ctypes as C
from contextlib import closing

import numpy as np
import pytest

from tests._oracle import make_grid, update_pairs
from tests.test_gpu_sharded_delta import _keys
from tests.test_oracle_delta import _cells

pytestmark = pytest.mark.gpu

DELTA_THREADS = 256
TBL_THREADS = 256
SCAN_TILE = 4096
LOOKBACK_HOP = 32
MS = 1_000_000
S0 = 0x10000
ID_SPACE = 1 << 21

A = dict(grid=(-5000.0, -5000.0, 100.0, 100.0, 100, 100), n0=400_000, grow=(2, 20_000), shrink=(4, 390_000), slots=160_000,
         radii=((20.0, 150.0), (400.0, 1500.0), 0.01), step=80.0, ticks=6, no_batch=3, fails=100, seed=11)
B = dict(grid=(-3000.0, -3000.0, 10.0, 10.0, 600, 600), n0=500_000, grow=None, shrink=None, slots=50_000,
         radii=((5.0, 40.0), (5.0, 40.0), 0.0), step=15.0, ticks=5, no_batch=None, fails=20, seed=12)


@pytest.fixture(scope="module")
def chd():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from channeld_b200 import capi, engine, synth

    capi.lib()

    class NS:
        pass

    ns = NS()
    ns.capi, ns.engine, ns.synth = capi, engine, synth
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ns.slot_warps = 32 * sms * DELTA_THREADS // 32  # delta_slots_kernel: warps of its largest grid
    ns.grid_threads = 8 * sms * DELTA_THREADS  # delta_moves / advance / id scatter kernels
    ns.tbl_threads = 8 * sms * TBL_THREADS  # tbl_delta_ids / commit kernels
    return ns


EMPTY = (np.zeros(0, np.uint32), np.zeros(1, np.uint64), np.zeros(0, np.uint32))  # no entities, no slots: the first snapshot


class Subscribers:
    """Per-slot query centres and radii; each tick a random 60 % of the slots query from a centre moved a little (so that most slots
    keep some cells and change others), and `fails` of those queries have radius 0 (they fail: the slot keeps its cells)."""

    def __init__(self, spec, rng):
        offx, offz, w, h, cols, rows = spec["grid"]
        self.lo, self.hi = (offx + 1.0, offz + 1.0), (offx + w * cols - 1.0, offz + h * rows - 1.0)
        S = spec["slots"]
        self.cx, self.cz = rng.uniform(self.lo[0], self.hi[0], S), rng.uniform(self.lo[1], self.hi[1], S)
        small, large, frac = spec["radii"]
        big = rng.random(S) < frac
        self.r = np.where(big, rng.uniform(*large, S), rng.uniform(*small, S))
        self.step, self.fails, self.S = 0.5 * w, spec["fails"], S

    def batch(self, rng):
        """-> (slots, cx, cz, r) of this tick's queries"""
        slots = np.nonzero(rng.random(self.S) < 0.6)[0]
        self.cx[slots] = np.clip(self.cx[slots] + rng.uniform(-self.step, self.step, len(slots)), self.lo[0], self.hi[0])
        self.cz[slots] = np.clip(self.cz[slots] + rng.uniform(-self.step, self.step, len(slots)), self.lo[1], self.hi[1])
        r = self.r[slots].copy()
        r[rng.choice(len(slots), self.fails, replace=False)] = 0.0
        return slots.astype(np.uint32), self.cx[slots].copy(), self.cz[slots].copy(), r


def _index_ticks(chd, spec):
    """The scripted world of case A or B, tick by tick -> (positions the engine sees, query batch or None).  Entities move with
    synth.move_entities; each tick about 3 % stand outside the world and 0.5 % are NaN (most come back); the array grows at the end on
    one tick and shrinks on another."""
    offx, offz, w, h, cols, rows = spec["grid"]
    rng = np.random.default_rng(spec["seed"])
    wc = chd.synth.WorldConfig("delta scale", offx, offz, w, h, cols, rows, 1, 1, spec["n0"], spec["slots"], 0.0, spec["seed"])
    x, z = offx + rng.random(spec["n0"]) * w * cols, offz + rng.random(spec["n0"]) * h * rows
    subs = Subscribers(spec, rng)
    for t in range(spec["ticks"]):
        if t:
            x, z = chd.synth.move_entities(wc, x, z, t, spec["step"])
        if spec["grow"] and t == spec["grow"][0]:
            k = spec["grow"][1]
            x, z = np.concatenate([x, offx + rng.random(k) * w * cols]), np.concatenate([z, offz + rng.random(k) * h * rows])
        if spec["shrink"] and t == spec["shrink"][0]:
            x, z = x[:spec["shrink"][1]], z[:spec["shrink"][1]]
        ex, ez = x.copy(), z.copy()
        out = rng.random(len(ex)) < 0.03
        ex[out] = offx - 1.0 - rng.random(out.sum()) * 100.0
        ez[rng.random(len(ez)) < 0.005] = np.nan
        yield ex, ez, (None if t == spec["no_batch"] else subs.batch(rng))


class Reference:
    """The pairs the engine keeps (from orc_sphere_tick without visible lists) and the oracle's state per tick."""

    def __init__(self, oracle, grid, n_slots):
        self.oracle, self.og, self.S = oracle, make_grid(*grid), n_slots
        self.cells = grid[4] * grid[5]
        self.off, self.pc = np.zeros(1, np.uint64), np.zeros(0, np.uint32)
        self.branches = dict(both=0, only_prev=0, only_now=0)

    def step(self, x, z, q):
        """-> (cell per entity, pair_off, pair_cell) after this tick's queries"""
        if q is not None:
            slots, cx, cz, r = q
            p = self.oracle.sphere_pairs(self.og, x, z, cx, cz, r)
            assert (p["status"][r > 0] == 0).all() and (p["status"][r == 0] != 0).all()
            off, pc = update_pairs(self.off, self.pc, self.S, slots, p["status"], p["pair_off"], p["pair_cell"].astype(np.int64) - S0)
            if len(self.off) == self.S + 1:  # cells a slot keeps (delta_side's moved-entity branch) and cells on one side only
                kp, kq = self._keys(self.off, self.pc), self._keys(off, pc)
                both = np.isin(kq, kp, assume_unique=True)
                self.branches["both"] += int(both.sum())
                self.branches["only_now"] += int((~both).sum())
                self.branches["only_prev"] += int((~np.isin(kp, kq, assume_unique=True)).sum())
            self.off, self.pc = off, pc
        return _cells(self.oracle, self.og, x, z), self.off, self.pc

    def _keys(self, off, pc):
        slot = np.repeat(np.arange(self.S, dtype=np.int64), np.diff(off.astype(np.int64)))
        return (slot << 32) | pc.astype(np.int64)


def _make_batch(chd, q):
    if q is None:
        return None, None
    slots, cx, cz, r = q
    return chd.engine.make_batch(len(slots), sub=slots, sphere=(cx, cz, r))


def _assert_exact(got, want, t):
    for name, u, v in zip(("enter_off", "enter", "leave_off", "leave"), got, want):
        np.testing.assert_array_equal(u, v, err_msg="tick %d %s" % (t, name))


def _assert_sets(got, want, n, t):
    """per slot the same entities (sorted slot << 32 | id keys), and no slot repeats an id"""
    for (go, ge), (wo, we), name in (((got[0], got[1]), (want[0], want[1]), "entered"), ((got[2], got[3]), (want[2], want[3]), "left")):
        kg, kw = _keys(go, ge, n), _keys(wo, we, n)
        assert (np.diff(kg) != 0).all(), (t, name)
        np.testing.assert_array_equal(kg, kw, err_msg="tick %d %s" % (t, name))


def _run_index_world(chd, oracle, spec, graphs=True, ids=False):
    """Cases A, B (index mode) and D (id mode: ids a random injection into [0, 2^21), the entity array permuted every tick)."""
    g = spec["grid"]
    C_ = g[4] * g[5]
    S = spec["slots"]
    n_max = spec["n0"] + (spec["grow"][1] if spec["grow"] else 0)
    ref = Reference(oracle, g, S)
    rng = np.random.default_rng(spec["seed"] + 100)
    gid = rng.choice(ID_SPACE, n_max, replace=False).astype(np.uint32)
    prev = EMPTY
    seen = dict(in_world=[], pairs=[], entered=0, left=0)
    with closing(chd.engine.Engine(chd.engine.grid_cfg(*g), n_max, S, max_pairs=1 << 22, max_window_cells=1 << 23)) as e:
        e.enable_graphs(graphs)
        e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
        if ids:
            e.reserve_visible_delta_ids(1 << 27, ID_SPACE)
        else:
            e.reserve_visible_delta(1 << 27)
        for t, (x, z, q) in enumerate(_index_ticks(chd, spec)):
            n = len(x)
            if ids:
                perm = rng.permutation(n)
                e.set_entities(x[perm], z[perm])
                e.set_entity_ids(gid[:n][perm])  # position i is entity perm[i]
            else:
                e.set_entities(x, z)
            batch, keep = _make_batch(chd, q)
            s = e.tick(batch, (t + 1) * 33 * MS, chd.capi.TICK_BUILD | chd.capi.TICK_VISIBLE_DELTA)
            assert s.overflow == 0
            now = ref.step(x, z, q)
            pairs = e.get_pairs()
            np.testing.assert_array_equal(pairs["off"].astype(np.uint64), now[1])
            np.testing.assert_array_equal(pairs["channel"] - S0, now[2])
            got = e.get_visible_delta()
            if ids:
                by_id = np.full(ID_SPACE, C_, np.uint32)
                by_id[gid[:n]] = now[0]  # each id takes the cell of its current position
                want = oracle.visible_delta(C_, prev, (by_id, now[1], now[2]))
                _assert_sets(got, want, S, t)
                prev = (by_id, now[1], now[2])
            else:
                want = oracle.visible_delta(C_, prev, now)
                _assert_exact(got, want, t)
                prev = now
            seen["in_world"].append(int((now[0] < C_).sum()))
            seen["empty_cells"] = C_ - len(np.unique(now[0][now[0] < C_]))
            seen["pairs"].append(len(now[2]))
            if t:
                seen["entered"] += len(got[1])
                seen["left"] += len(got[3])
    return seen, ref.branches


def _assert_common(seen, branches):
    assert seen["entered"] > 0 and seen["left"] > 0
    assert min(branches.values()) > 0, branches  # both branches of delta_side, on both sides


@pytest.mark.parametrize("graphs", [True, False], ids=["graphs", "direct"])
def test_a_many_slots(chd, oracle, graphs):
    seen, branches = _run_index_world(chd, oracle, A, graphs)
    _assert_common(seen, branches)
    assert A["slots"] > chd.slot_warps and A["slots"] > LOOKBACK_HOP * SCAN_TILE
    assert min(seen["in_world"]) > chd.grid_threads, (seen["in_world"], chd.grid_threads)
    assert min(seen["pairs"][1:]) > chd.grid_threads, (seen["pairs"], chd.grid_threads)


def test_b_many_cells(chd, oracle):
    C_ = B["grid"][4] * B["grid"][5]
    assert C_ + 1 > chd.grid_threads, (C_, chd.grid_threads)
    seen, branches = _run_index_world(chd, oracle, B)
    _assert_common(seen, branches)
    assert seen["empty_cells"] > C_ // 10, seen["empty_cells"]


def test_d_id_mode(chd, oracle):
    seen, branches = _run_index_world(chd, oracle, A, ids=True)
    _assert_common(seen, branches)
    assert A["slots"] > chd.slot_warps
    assert A["n0"] > chd.grid_threads and min(seen["in_world"]) > chd.grid_threads


def test_c_benchmark_world_beside_the_full_tick(chd, oracle):
    """bench_visible_delta.py's workload with TICK_ALL | TICK_VISIBLE_DELTA: the emit and fan-out run beside the delta."""
    L = chd.capi.lib()
    wc = chd.synth.CONFIGS["benchmark"]
    N, S = wc.n_entities, wc.n_subscribers
    assert S > chd.slot_warps and N > chd.grid_threads
    og = make_grid(wc.offx, wc.offz, wc.w, wc.h, wc.cols, wc.rows, wc.server_cols, wc.server_rows)
    x, z = chd.synth.entities(wc)
    idx = (np.arange(S, dtype=np.int64) * (N // S)) % N
    r = np.full(S, wc.radius)
    prev, ring_state = None, None
    with closing(chd.engine.Engine(wc.cfg(), N, S)) as e:
        e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
        e.reserve_visible_delta(600_000_000)  # the first delta enters every visible list
        for t in range(4):
            if t:
                x, z = chd.synth.move_entities(wc, x, z, t, 60.0)
            ring_state, off, arr, snd, ridx, cmi = chd.synth.update_rings(wc, t, (t + 1) * 33 * MS, 33 * MS, 4, S, ring_len=64, state=ring_state)
            e.set_entities(x, z)
            e.set_rings(off, arr, snd, ridx, cmi)
            batch, keep = chd.engine.make_batch(S, sub=np.arange(S, dtype=np.uint32), sphere=(x[idx].copy(), z[idx].copy(), r))
            s = e.tick(batch, (t + 1) * 33 * MS, chd.capi.TICK_ALL | chd.capi.TICK_VISIBLE_DELTA)
            assert s.overflow == 0
            p = oracle.sphere_pairs(og, x, z, x[idx], z[idx], r)
            assert (p["status"] == 0).all()
            now = (_cells(oracle, og, x, z), p["pair_off"], (p["pair_cell"].astype(np.int64) - S0).astype(np.uint32))
            assert int((now[0] < wc.cells).sum()) > chd.grid_threads
            if t == 0:  # the whole visible list (about 4.9e8 entries): offsets only
                eo, lo, voff = np.zeros(S + 1, np.uint64), np.zeros(S + 1, np.uint64), np.zeros(S + 1, np.uint64)
                ne, nl, ns = C.c_uint64(), C.c_uint64(), C.c_uint32()
                assert L.chd_get_visible_delta(e.h, chd.capi.ptr(eo), None, chd.capi.ptr(lo), None, 0, C.byref(ne), C.byref(nl), C.byref(ns)) == 0
                assert L.chd_get_visible(e.h, chd.capi.ptr(voff), None) == 0
                assert ns.value == S and nl.value == 0 and not lo.any()
                np.testing.assert_array_equal(eo, voff)
                np.testing.assert_array_equal(eo, p["vis_off"])
                assert ne.value == s.n_visible > 1e8
            else:
                got = e.get_visible_delta()
                want = oracle.visible_delta(wc.cells, prev, now)
                _assert_exact(got, want, t)
                assert len(got[1]) > 1e7 and len(got[3]) > 1e7
            prev = now


def test_e_entity_table_mode(chd, oracle):
    """400 K ids spawned once (table slots are handed out in spawn order), 30 % of them moved per tick; the reference is the
    index-mode oracle over table slots, named through slot -> id.  No despawns: test_gpu_entity_table covers despawn and quarantine."""
    spec = dict(A, ticks=5)
    g = spec["grid"]
    offx, offz, w, h, cols, rows = g
    C_ = cols * rows
    N, S = spec["n0"], spec["slots"]
    assert N > chd.tbl_threads and N > chd.grid_threads and S > chd.slot_warps
    rng = np.random.default_rng(21)
    ids = (rng.choice((1 << 31) - 1, N, replace=False) + 1).astype(np.uint32)  # 31-bit, never a reserved id
    x, z = offx + rng.random(N) * w * cols, offz + rng.random(N) * h * rows
    wc = chd.synth.WorldConfig("delta scale table", offx, offz, w, h, cols, rows, 1, 1, N, S, 0.0, 21)
    subs = Subscribers(spec, rng)
    ref = Reference(oracle, g, S)
    prev = EMPTY
    entered = []
    with closing(chd.engine.Engine(chd.engine.grid_cfg(*g), N, S, max_pairs=1 << 22, max_window_cells=1 << 23)) as e:
        e.entity_table_init()
        e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
        e.reserve_visible_delta(1 << 27)
        assert (e.spawn_entities(ids, x, z) == chd.capi.EV_OK).all()
        for t in range(spec["ticks"]):
            if t:  # 30 % move; a few of them step outside the world, and some come back
                mv = np.sort(rng.choice(N, 3 * N // 10, replace=False))
                nx, nz = chd.synth.move_entities(wc, x[mv], z[mv], t, 150.0)
                nx[rng.random(len(mv)) < 0.05] = offx - 10.0
                x[mv], z[mv] = nx, nz
                e.move_entities(ids[mv], nx, nz)
            q = subs.batch(rng)
            batch, keep = _make_batch(chd, q)
            s = e.tick(batch, (t + 1) * 33 * MS, chd.capi.TICK_BUILD | chd.capi.TICK_VISIBLE_DELTA)
            assert s.overflow == 0
            now = ref.step(x, z, q)
            assert e.entity_stats()["high_water"] == N
            want = oracle.visible_delta(C_, prev, now)
            got = e.get_visible_delta()
            # index mode's order (cell, then table slot) translated to ids: exact
            _assert_exact(got, (want[0], ids[want[1]], want[2], ids[want[3]]), t)
            entered.append(len(got[1]))
            prev = now
    assert entered[0] > chd.tbl_threads, (entered, chd.tbl_threads)
    assert min(ref.branches.values()) > 0, ref.branches
