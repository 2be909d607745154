"""Numpy restatements of the X-slab building blocks (include/chd_gpu.h, multi-GPU X-slab sharding; chd_shard.cuh): which own
entities a slab exports, which gathered records it imports, which own entities it re-homes, and which emit kernel it takes.
Written from the documented rules, not from the kernels, so that tests can hold the kernels to them.  CPU only."""
import numpy as np

from channeld_b200 import sharding

EMIT_TILE = 2048  # CTA emit tile (chd_types.cuh)


def grid_cells(x, z, offx, offz, w, h, cols, rows):
    """Cell index col + row * cols of each position, -1 outside the world: floor((x - offx) / w) in f64, one rounding per
    operation, as GetChannelIdWithOffset computes it."""
    fx = np.floor((np.asarray(x, np.float64) - offx) / w)
    fz = np.floor((np.asarray(z, np.float64) - offz) / h)
    ok = (fx >= 0) & (fx < cols) & (fz >= 0) & (fz < rows)
    return np.where(ok, np.where(ok, fx, 0) + np.where(ok, fz, 0) * cols, -1).astype(np.int64)


def export_set(cell, gid, cols, col_lo, col_hi, halo):
    """Records (gid, cell) a slab [col_lo, col_hi) exports, in entity order: own in-world entities whose column is not strictly
    interior (within `halo` columns of a slab edge), except on a side where the slab ends at the world's edge, plus every own
    in-world entity that left the slab."""
    cell = np.asarray(cell, np.int64)
    col = np.where(cell >= 0, cell % cols, -1)
    in_world = cell >= 0
    left = col < col_lo + halo          # within halo columns of the left edge
    right = col >= col_hi - halo        # within halo columns of the right edge
    interior = ~left & ~right
    closed_left_only = left & ~right & (col_lo == 0)
    closed_right_only = right & ~left & (col_hi == cols)
    closed_both = left & right & (col_lo == 0) & (col_hi == cols)
    left_slab = (col < col_lo) | (col >= col_hi)
    keep = in_world & (left_slab | (~interior & ~closed_left_only & ~closed_right_only & ~closed_both))
    return np.asarray(gid, np.int64)[keep], cell[keep]


def served_columns(cols, col_lo, col_hi, halo):
    """[a, b): the columns a slab serves, clipped to the world"""
    return max(0, col_lo - halo), min(cols, col_hi + halo)


def import_set(records, rank, cols, cells, col_lo, col_hi, halo):
    """records[r] = (gid, cell) exported by rank r.  -> (gid, cell, src_rank) of the records `rank` keeps, in gathered order:
    every other rank's records whose cell is in the world and lies in a served column."""
    a, b = served_columns(cols, col_lo, col_hi, halo)
    out = [], [], []
    for r, (g, c) in enumerate(records):
        if r == rank:
            continue
        c = np.asarray(c, np.int64)
        keep = (c >= 0) & (c < cells) & (c % cols >= a) & (c % cols < b)
        out[0].append(np.asarray(g, np.int64)[keep])
        out[1].append(c[keep])
        out[2].append(np.full(int(keep.sum()), r, np.int64))
    return tuple(np.concatenate(o) if o else np.zeros(0, np.int64) for o in out)


def rehome_set(cell, gid, cols, col_lo, col_hi, world):
    """(gid, destination rank) of the own in-world entities whose column lies outside [col_lo, col_hi)"""
    cell = np.asarray(cell, np.int64)
    col = cell % cols
    away = (cell >= 0) & ((col < col_lo) | (col >= col_hi))
    return np.asarray(gid, np.int64)[away], sharding.owner_of_column(col[away], cols, world)


def emit_uses_cta_tiles(n_own, slab_cols, rows, n_build, l2_bytes):
    """The emit kernel a slab takes: CTA tiles when its own entities average at least EMIT_TILE / 2 per own cell and its build
    (own + border capacity; 0 for an engine without chd_comm_init) fits L2 / 32 at 16 bytes an entity; warp tiles otherwise."""
    return n_own // max(slab_cols * rows, 1) >= EMIT_TILE // 2 and n_build * 16 <= l2_bytes // 2


def boundary_xs(offx, w, cols, slabs, halo):
    """x = offx + k * w and its f64 neighbours on either side, for k in {0, cols} and every slab's col_lo, col_hi, col_lo +- halo
    and col_hi +- halo.  -> (x, k)"""
    ks = {0, cols}
    for lo, hi in slabs:
        ks |= {lo, hi, lo - halo, lo + halo, hi - halo, hi + halo}
    xs, kk = [], []
    for k in sorted(ks):
        x0 = offx + k * w
        for x in (np.nextafter(x0, -np.inf), x0, np.nextafter(x0, np.inf)):
            xs.append(x)
            kk.append(k)
    return np.array(xs, np.float64), np.array(kk, np.int64)


def keys(gid, cell):
    """(gid, cell) records as sorted u64 keys cell << 32 | gid: a multiset to compare"""
    return np.sort((np.asarray(cell, np.int64).astype(np.uint64) << np.uint64(32)) | np.asarray(gid, np.int64).astype(np.uint64))
