"""Random SpatialInterestQuery batches in chd_query_batch's layout (engine.make_batch's keyword arguments), aimed at the edges of
QueryChannelIds (spatial.go:182-317), and a numpy restatement of the kernel's per-query cell window (query_bbox, chd_query.cuh).
Test infrastructure: no GPU needed."""
import math

import numpy as np

AOI_SPOTS, AOI_BOX, AOI_SPHERE, AOI_CONE = 1, 2, 4, 8


def _pick(rng, n, choices, p):
    """choices: arrays of n values (or scalars); row i takes choices[k][i] with probability p[k]"""
    k = rng.choice(len(choices), size=n, p=np.asarray(p, float) / np.sum(p))
    out = np.zeros(n)
    for j, c in enumerate(choices):
        m = k == j
        out[m] = np.broadcast_to(np.asarray(c, np.float64), (n,))[m]
    return out


def _reach(rng, n, w, h, long_cells):
    """radii / extents: below a cell, a few cells, exact multiples of the cell size (samples on cell edges), and now and then a
    reach of `long_cells` cells (windows of 1000+ cells)"""
    cell, mn = max(w, h), min(w, h)
    k = rng.integers(1, 5, n).astype(np.float64)
    return _pick(rng, n, [rng.uniform(0.01, 0.45, n) * mn, rng.uniform(0.5, 3.0, n) * cell, k * w, k * h, k * 0.5 * w,
                          rng.uniform(0.8, 1.2, n) * long_cells * cell],
                 [0.3, 0.3, 0.12, 0.12, 0.1, 0.03])


def make_queries(rng, grid, n, cx=None, cz=None, kind=None, p_err=0.03, long_cells=20.0, max_spots=300):
    """-> dict(n, kind, sphere, box, cone, spots) for engine.make_batch(n, **q) and Oracle.query_batch(og, **q).
    grid = (offx, offz, w, h, cols, rows).  kind: all 16 masks uniformly unless given; cx / cz: the query centres (random in the
    world unless given, a quarter of them on exact cell corners).  A share p_err of the queries with a shape takes an error path:
    centre out of the world, radius / extent <= 0, an absorbed step (v + step == v), or a cone angle of 2^29."""
    offx, offz, w, h, cols, rows = grid
    ww, wh = w * cols, h * rows
    if kind is None:
        kind = rng.integers(0, 16, n)
    kind = np.asarray(kind, np.uint8)
    if cx is None:
        cx = offx + rng.uniform(0, 1, n) * ww
        cz = offz + rng.uniform(0, 1, n) * wh
        snap = rng.random(n) < 0.25  # exact multiples of the cell size: samples land on cell edges
        cx[snap] = offx + w * rng.integers(0, cols, snap.sum())
        cz[snap] = offz + h * rng.integers(0, rows, snap.sum())
    cx, cz = np.asarray(cx, np.float64).copy(), np.asarray(cz, np.float64).copy()
    xmax, zmax = np.nextafter(offx + ww, -np.inf), np.nextafter(offz + wh, -np.inf)

    # sphere
    sr = _reach(rng, n, w, h, long_cells)
    # box: its own centre near the sphere's, extents drawn independently; some long and thin (a whole row band / column band)
    bx = np.clip(cx + rng.uniform(-0.6, 0.6, n) * w * (rng.random(n) < 0.5), offx, xmax)
    bz = np.clip(cz + rng.uniform(-0.6, 0.6, n) * h * (rng.random(n) < 0.5), offz, zmax)
    bex, bez = _reach(rng, n, w, h, long_cells), _reach(rng, n, w, h, long_cells)
    thin = rng.random(n)
    bex[thin < 0.03] = rng.uniform(0.2, 0.35, (thin < 0.03).sum()) * ww
    bez[thin < 0.03] = rng.uniform(0.2, 1.5, (thin < 0.03).sum()) * h
    bez[thin > 0.97] = rng.uniform(0.2, 0.35, (thin > 0.97).sum()) * wh
    bex[thin > 0.97] = rng.uniform(0.2, 1.5, (thin > 0.97).sum()) * w
    # cone: at the world's edge for a third, angles 0, pi/4, just below pi and random; some axis-aligned directions
    # (the largest double below the world's max edge is in the world only where subtracting the offset keeps it below: now and then)
    ccx, ccz = cx.copy(), cz.copy()
    edge = rng.integers(0, 48, n)
    ccx[edge < 8], ccx[(edge >= 8) & (edge < 16)] = offx, offx + ww * (1 - 1e-9)
    ccz[(edge >= 16) & (edge < 24)], ccz[(edge >= 24) & (edge < 32)] = offz, offz + wh * (1 - 1e-9)
    ccx[edge == 32], ccz[edge == 33] = xmax, zmax
    ang = rng.uniform(0, 2 * math.pi, n)
    cdx, cdz = np.cos(ang), np.sin(ang)
    axis = rng.integers(0, 8, n)
    cdx[axis == 0], cdz[axis == 0] = 1.0, 0.0
    cdx[axis == 1], cdz[axis == 1] = 0.0, -1.0
    cangle = _pick(rng, n, [0.0, math.pi / 4, np.nextafter(math.pi, 0), rng.uniform(0, 3.2, n), 0.5236], [0.15, 0.25, 0.15, 0.35, 0.1])
    cr = _reach(rng, n, w, h, long_cells)

    # error paths, one per chosen query, on a shape it has
    err = (rng.random(n) < p_err) & ((kind & (AOI_BOX | AOI_SPHERE | AOI_CONE)) != 0)
    for i in np.nonzero(err)[0]:
        shapes = [b for b in (AOI_BOX, AOI_SPHERE, AOI_CONE) if kind[i] & b]
        b = shapes[rng.integers(0, len(shapes))]
        how = rng.integers(0, 4 if b == AOI_CONE else 3)
        if how == 0:  # centre out of the world
            ox, oz = offx + rng.choice([-0.3, 1.0, 1.3]) * ww, offz + rng.uniform(0, 1) * wh
            if b == AOI_BOX:
                bx[i], bz[i] = ox, oz
            elif b == AOI_SPHERE:
                cx[i], cz[i] = ox, oz
            else:
                ccx[i], ccz[i] = ox, oz
        elif how == 1:  # radius / extent <= 0
            v = rng.choice([0.0, -1.0, -0.0])
            if b == AOI_BOX:
                if rng.random() < 0.5:
                    bex[i] = v
                else:
                    bez[i] = v
            elif b == AOI_SPHERE:
                sr[i] = v
            else:
                cr[i] = v
        elif how == 2:  # absorbed step: the reference would never terminate
            if b == AOI_BOX:
                bx[i], bex[i], bez[i] = 1e17, 1.0, 1.0
            elif b == AOI_SPHERE:
                cx[i], sr[i] = 1e17, 1.0
            else:
                ccx[i], cr[i] = -1e17, 1.0
        else:
            cangle[i] = float(1 << 29)

    # spots: 1-6 per query mostly, up to max_spots; outside the world, next to the sphere's centre (same rows: side cells that
    # interleave with the window), repeated cells with different dists; len(Dists) below, equal to and above len(Spots)
    has = (kind & AOI_SPOTS) != 0
    cnt = np.zeros(n, np.int64)
    m = int(has.sum())
    cnt[has] = _pick(rng, m, [rng.integers(1, 7, m), rng.integers(7, 65, m), rng.integers(65, max_spots + 1, m)], [0.75, 0.17, 0.08])
    off = np.concatenate([[0], np.cumsum(cnt)]).astype(np.uint32)
    T = int(off[-1])
    owner = np.repeat(np.arange(n), cnt)
    mode = rng.choice(4, size=T, p=[0.55, 0.25, 0.1, 0.1])
    sx = offx + rng.uniform(-0.05, 1.05, T) * ww
    sz = offz + rng.uniform(-0.05, 1.05, T) * wh
    near = mode == 1
    sx[near] = cx[owner[near]] + rng.integers(-12, 13, near.sum()) * w + rng.uniform(0, 0.9, near.sum()) * w
    sz[near] = cz[owner[near]] + rng.uniform(-1.5, 1.5, near.sum()) * h
    edge_ = mode == 2  # on cell corners, some on the world's max edge (outside)
    sx[edge_] = offx + w * rng.integers(0, cols + 1, edge_.sum())
    sz[edge_] = offz + h * rng.integers(0, rows + 1, edge_.sum())
    first = np.zeros(T, bool)
    first[off[:-1][cnt > 0]] = True
    dup = np.nonzero((mode == 3) & ~first)[0]  # the previous spot's cell again (last write wins)
    for j in dup:  # in order, so a run of repeats copies one position
        sx[j], sz[j] = sx[j - 1] + 0.25 * w * rng.random(), sz[j - 1]
    sd = _pick(rng, T, [rng.integers(0, 6, T), 3, 1000, 2 ** 31, 0xFFFFFFFE], [0.75, 0.05, 0.1, 0.05, 0.05]).astype(np.uint32)
    nd_mode = rng.integers(0, 3, n)
    nd = np.where(nd_mode == 0, (rng.random(n) * cnt).astype(np.int64), np.where(nd_mode == 1, cnt, cnt + rng.integers(1, 4, n)))
    return dict(n=n, kind=kind, sphere=(cx, cz, sr), box=(bx, bz, bex, bez), cone=(ccx, ccz, cdx, cdz, cangle, cr),
                spots=(off, nd.astype(np.uint32), sx, sz, sd))


def take(q, idx):
    """The queries idx of a batch (a new batch, in that order)."""
    idx = np.asarray(idx, np.int64)
    off, nd, sx, sz, sd = q["spots"]
    cnt = np.diff(off.astype(np.int64))[idx]
    noff = np.concatenate([[0], np.cumsum(cnt)]).astype(np.uint32)
    src = np.repeat(off[:-1].astype(np.int64)[idx] - noff[:-1], cnt) + np.arange(int(noff[-1]))
    return dict(n=len(idx), kind=q["kind"][idx], sphere=tuple(a[idx] for a in q["sphere"]), box=tuple(a[idx] for a in q["box"]),
                cone=tuple(a[idx] for a in q["cone"]), spots=(noff, nd[idx], sx[src], sz[src], sd[src]))


def batch_kwargs(q):
    return {k: v for k, v in q.items() if k != "n"}


# ---------------------------------------------------------------- the kernel's cell window, restated

def _go_min(x, y):
    r = np.minimum(x, y)  # NaN-propagating
    return np.where(np.isneginf(x), x, np.where(np.isneginf(y), y, r))


def _go_max(x, y):
    r = np.maximum(x, y)
    return np.where(np.isposinf(x), x, np.where(np.isposinf(y), y, r))


def grid_coord(grid, x, z):
    """-> (valid, gx, gy): floor((v - off) / w) tested in double before the conversion, as grid_coord / cell_index do"""
    offx, offz, w, h, cols, rows = grid
    with np.errstate(invalid="ignore", over="ignore"):
        fx = np.floor((np.asarray(x, np.float64) - offx) / w)
        fz = np.floor((np.asarray(z, np.float64) - offz) / h)
        ok = (fx >= 0) & (fx < float(cols)) & (fz >= 0) & (fz < float(rows))
    return ok, np.where(ok, fx, 0).astype(np.int64), np.where(ok, fz, 0).astype(np.int64)


def query_windows(grid, q):
    """query_bbox for every query: -> (gx0, gy0, bw, bh) int64 arrays; bw = bh = 0 for an empty window.  The box spans the
    columns / rows of each shape's first and last lattice coordinate (a cone's clamped to the world) plus each shape's centre
    cell, with the kernel's IEEE operations (subtract, divide, floor, compare, clamp)."""
    offx, offz, w, h, cols, rows = grid
    n = q["n"]
    kind = q["kind"].astype(np.int64)
    fcols, frows = float(cols), float(rows)
    x0 = np.full(n, np.iinfo(np.int64).max); y0 = x0.copy()
    x1 = np.full(n, -1, np.int64); y1 = x1.copy()

    def add(m, a0, a1, b0, b1):
        np.minimum(x0, np.where(m, a0, x0), out=x0); np.maximum(x1, np.where(m, a1, x1), out=x1)
        np.minimum(y0, np.where(m, b0, y0), out=y0); np.maximum(y1, np.where(m, b1, y1), out=y1)

    def add_range(m, xlo, xhi, zlo, zhi):
        with np.errstate(invalid="ignore", over="ignore"):
            m = m & (xlo <= xhi) & (zlo <= zhi)
            fl, fh = np.floor((xlo - offx) / w), np.floor((xhi - offx) / w)
            rl, rh = np.floor((zlo - offz) / h), np.floor((zhi - offz) / h)
            m = m & (fh >= 0) & (fl < fcols) & (rh >= 0) & (rl < frows)
            a0 = np.where(fl < 0, 0, np.where(m, fl, 0)).astype(np.int64)
            a1 = np.where(fh >= fcols, cols - 1, np.where(m, fh, 0)).astype(np.int64)
            b0 = np.where(rl < 0, 0, np.where(m, rl, 0)).astype(np.int64)
            b1 = np.where(rh >= frows, rows - 1, np.where(m, rh, 0)).astype(np.int64)
        add(m, a0, a1, b0, b1)

    def add_point(m, x, z):
        ok, gx, gy = grid_coord(grid, x, z)
        add(m & ok, gx, gx, gy, gy)

    m = (kind & AOI_BOX) != 0
    cx, cz, ex, ez = q["box"]
    add_range(m, cx - ex, cx + ex, cz - ez, cz + ez)
    add_point(m, cx, cz)
    m = (kind & AOI_SPHERE) != 0
    cx, cz, r = q["sphere"][:3]
    add_range(m, cx - r, cx + r, cz - r, cz + r)
    add_point(m, cx, cz)
    m = (kind & AOI_CONE) != 0
    cx, cz, r = q["cone"][0], q["cone"][1], q["cone"][5]
    wxh, wzh = offx + w * fcols, offz + h * frows
    add_range(m, _go_max(offx, cx - r), _go_min(wxh, cx + r), _go_max(offz, cz - r), _go_min(wzh, cz + r))
    add_point(m, cx, cz)
    anyc = x1 >= 0
    gx0, gy0 = np.where(anyc, x0, 0), np.where(anyc, y0, 0)
    bw, bh = np.where(anyc, x1 - x0 + 1, 0), np.where(anyc, y1 - y0 + 1, 0)
    return gx0, gy0, bw, bh
