"""The oracle's visible-set delta (orc_visible_delta) against set differences of consecutive orc_sphere_tick visible lists, on small
worlds whose entities leave the world, turn NaN, and are added or removed at the end of the array, whose slot count grows, and
whose slots send failing queries or none at all.  No GPU needed."""
import ctypes as C

import numpy as np
import pytest

from tests._oracle import ERR_CAPACITY, make_grid, update_pairs
from tests.test_gpu_visible_delta import _set_diff

S0 = 0x10000
GRIDS = {  # offx, offz, w, h, cols, rows
    "10x8": (-500.0, -400.0, 100.0, 100.0, 10, 8),
    "2x2": (-2000.0, -2000.0, 2000.0, 2000.0, 2, 2),
}
RADII = {"10x8": (20.0, 350.0), "2x2": (50.0, 2500.0)}


def _cells(oracle, og, x, z):
    """cell index per entity, the cell count for one outside the world (or NaN)"""
    c = oracle.cell_of(og, x, z).astype(np.int64) - S0
    return np.where(c < 0, og.grid_cols * og.grid_rows, c).astype(np.uint32)


def _script(rng, name, n_ticks):
    """per tick: entity positions and, for a growing slot count, the query batch (slots, cx, cz, r) of that tick"""
    offx, offz, w, h, cols, rows = GRIDS[name]
    W, H = w * cols, h * rows
    n = 3000
    x, z = offx + rng.random(n) * W, offz + rng.random(n) * H
    lo, hi = RADII[name]
    for t in range(n_ticks):
        n_slots = 40 + 10 * min(t, 3)  # grows on ticks 1 to 3
        if t:
            step = rng.uniform(-0.4, 0.4, (2, len(x))) * w
            x, z = x + step[0], z + step[1]
            if t == 2:  # added at the end of the array
                x = np.concatenate([x, offx + rng.random(400) * W])
                z = np.concatenate([z, offz + rng.random(400) * H])
            if t == 4:  # removed from the end
                x, z = x[:2500], z[:2500]
        px, pz = x.copy(), z.copy()
        out = rng.random(len(px)) < 0.04  # outside the world this tick (some come back later)
        px[out] = offx - 10.0 - rng.random(out.sum()) * W
        px[rng.random(len(px)) < 0.02] = np.nan
        # slots 0..4 never query (empty); the others query at random; a few queries fail (radius 0, centre outside the world)
        slots = np.nonzero(rng.random(n_slots) < 0.6)[0]
        slots = slots[slots >= 5].astype(np.uint32)
        cx, cz = offx + rng.random(len(slots)) * W, offz + rng.random(len(slots)) * H
        r = rng.uniform(lo, hi, len(slots))
        bad = rng.random(len(slots)) < 0.08
        r[bad & (rng.random(len(slots)) < 0.5)] = 0.0
        cx[bad & (r > 0)] = offx - 5.0
        yield px, pz, n_slots, (slots, cx, cz, r)


@pytest.mark.parametrize("grid", list(GRIDS))
def test_delta_oracle_is_the_set_difference_of_visible_lists(oracle, grid):
    g = GRIDS[grid]
    og = make_grid(*g)
    Cn = g[4] * g[5]
    rng = np.random.default_rng(5 + Cn)
    # the query in effect per slot: radius 0 fails, so a slot that never queried has no cells
    eff = np.zeros((3, 0))
    prev_vis = (np.zeros(1, np.uint64), np.zeros(0, np.uint32))
    prev = (np.zeros(0, np.uint32), np.zeros(1, np.uint64), np.zeros(0, np.uint32))  # the empty snapshot
    kinds = dict(entered=0, left=0, failed=0, both=0, only_p=0, only_q=0)
    for t, (x, z, n_slots, (slots, cx, cz, r)) in enumerate(_script(rng, grid, 7)):
        eff = np.concatenate([eff, np.array([[g[0] - 1.0], [g[1] - 1.0], [0.0]]).repeat(n_slots - eff.shape[1], 1)], axis=1)
        q = oracle.sphere_pairs(og, x, z, cx, cz, r)
        ok = q["status"] == 0
        kinds["failed"] += int((~ok).sum())
        eff[:, slots[ok]] = np.stack([cx[ok], cz[ok], r[ok]])
        want = oracle.sphere_tick(og, x, z, eff[0], eff[1], eff[2])
        # the pairs the engine keeps (a failed query keeps the slot's cells) are the effective queries' pairs
        off, pc = update_pairs(prev[1], prev[2], n_slots, slots, q["status"], q["pair_off"], q["pair_cell"].astype(np.int64) - S0)
        np.testing.assert_array_equal(off, want["pair_off"])
        np.testing.assert_array_equal(pc, want["pair_cell"] - S0)
        now = (_cells(oracle, og, x, z), off, pc)
        got = oracle.visible_delta(Cn, prev, now)
        vis = (want["vis_off"], want["vis_entity"])
        exp = _set_diff(prev_vis, vis, n_slots)
        for u, v in zip(got, exp):
            np.testing.assert_array_equal(u, v)
        kinds["entered"] += len(got[1])
        kinds["left"] += len(got[3])
        if t:  # cells a slot had before and has now, and cells on one side only
            def keys(o, c):
                o = np.concatenate([o.astype(np.int64), np.full(n_slots + 1 - len(o), int(o[-1]))])
                return np.repeat(np.arange(n_slots, dtype=np.int64), np.diff(o)) << 32 | c.astype(np.int64)

            kp, kq = keys(prev[1], prev[2]), keys(off, pc)
            kinds["both"] += int(np.isin(kq, kp).sum())
            kinds["only_p"] += int((~np.isin(kp, kq)).sum())
            kinds["only_q"] += int((~np.isin(kq, kp)).sum())
        prev, prev_vis = now, vis
    assert all(v > 0 for v in kinds.values()), kinds


def test_delta_oracle_counts_alone_and_refuses_a_short_buffer(oracle):
    g = GRIDS["10x8"]
    og = make_grid(*g)
    rng = np.random.default_rng(3)
    x, z = g[0] + rng.random(500) * 1000, g[1] + rng.random(500) * 800
    cx, cz = g[0] + rng.random(20) * 1000, g[1] + rng.random(20) * 800
    q = oracle.sphere_pairs(og, x, z, cx, cz, np.full(20, 150.0))
    now = (_cells(oracle, og, x, z), q["pair_off"], (q["pair_cell"] - S0).astype(np.uint32))
    empty = (np.zeros(0, np.uint32), np.zeros(1, np.uint64), np.zeros(0, np.uint32))
    eo, en, lo, le = oracle.visible_delta(og.grid_cols * og.grid_rows, empty, now)
    np.testing.assert_array_equal(eo, q["vis_off"])
    assert len(le) == 0 and len(en) > 10
    # everything leaves when the roles swap
    lo2 = oracle.visible_delta(og.grid_cols * og.grid_rows, now, empty)[2]
    np.testing.assert_array_equal(lo2, eo)
    # a buffer one entry short: ORC_ERR_CAPACITY, nothing written
    u32p, u64p = C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)
    cell, off, pc = (np.ascontiguousarray(a) for a in now)
    out_e, out_l = np.full(len(en), 7, np.uint32), np.zeros(1, np.uint32)
    eo2, lo3 = np.zeros(21, np.uint64), np.zeros(21, np.uint64)
    e0, o0, c0 = np.zeros(1, np.uint32), np.zeros(1, np.uint64), np.zeros(1, np.uint32)
    p = lambda a, t: a.ctypes.data_as(t)  # noqa: E731
    rc = oracle.lib.orc_visible_delta(og.grid_cols * og.grid_rows, p(e0, u32p), 0, p(o0, u64p), p(c0, u32p), 0, p(cell, u32p), len(cell),
                                      p(off, u64p), p(pc, u32p), 20, p(eo2, u64p), p(out_e, u32p), len(en) - 1, p(lo3, u64p), p(out_l, u32p),
                                      1, 2)
    assert rc == ERR_CAPACITY
    assert (out_e == 7).all()
    np.testing.assert_array_equal(eo2, eo)
