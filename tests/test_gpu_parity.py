"""GPU parity tests: the CUDA path, called through the C ABI, against the CPU oracle on the same inputs.
Bit-exact: integer/index work, and FP64 work that must reproduce Go's rounding operation by operation.
Run on an H100:  python -m pytest tests -m gpu
"""
import ctypes as C
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

S0 = 65536
MS = 1_000_000


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


def _ctl(chd, offx, offz, w, h, cols, rows, scols=1, srows=1, border=0):
    c = chd.controller.GpuStaticGrid2DSpatialController(max_entities=4096, max_subscribers=256)
    c.LoadConfig(dict(WorldOffsetX=offx, WorldOffsetZ=offz, GridWidth=w, GridHeight=h, GridCols=cols, GridRows=rows,
                      ServerCols=scols, ServerRows=srows, ServerInterestBorderSize=border))
    return c


def _sphere(cx, cz, r):
    C = __import__("channeld_b200.controller", fromlist=["x"])
    return C.SpatialInterestQuery(SphereAOI=C.SphereAOI(Center=C.SpatialInfo(X=cx, Z=cz), Radius=r))


def _box(cx, cz, ex, ez):
    C = __import__("channeld_b200.controller", fromlist=["x"])
    return C.SpatialInterestQuery(BoxAOI=C.BoxAOI(Center=C.SpatialInfo(X=cx, Z=cz), Extent=C.SpatialInfo(X=ex, Z=ez)))


def _cone(cx, cz, dx, dz, angle, r):
    C = __import__("channeld_b200.controller", fromlist=["x"])
    return C.SpatialInterestQuery(ConeAOI=C.ConeAOI(Center=C.SpatialInfo(X=cx, Z=cz), Direction=C.SpatialInfo(X=dx, Z=dz),
                                                    Angle=angle, Radius=r))


# ----------------------------------------------------------------- the reference's own KATs, through the C ABI

def test_kat_get_channel_id(chd):  # spatial_test.go:762-848
    SI, SE = chd.controller.SpatialInfo, chd.controller.SpatialError
    c = _ctl(chd, -450, -200, 100, 50, 9, 8, 3, 4, 2)
    assert c.GetChannelId(SI(X=-450, Z=-200)) == S0
    assert c.GetChannelId(SI(X=-350, Z=-200)) == S0 + 1
    assert c.GetChannelId(SI(X=-450, Z=-150)) == S0 + 9
    assert c.GetChannelId(SI(X=0, Z=0)) == S0 + 9 * 4 + 4
    assert c.GetChannelId(SI(X=449.99, Z=199.99)) == S0 + 9 * 8 - 1
    for x, z in [(-500, 0), (500, 0), (0, -300), (0, 300), (450, 200)]:
        with pytest.raises(SE):
            c.GetChannelId(SI(X=x, Z=z))
    c = _ctl(chd, 0, 0, 100, 50, 9, 8, 3, 4, 2)
    assert c.GetChannelId(SI(X=0, Z=0)) == S0
    assert c.GetChannelId(SI(X=100, Z=0)) == S0 + 1
    assert c.GetChannelId(SI(X=0, Z=50)) == S0 + 9
    assert c.GetChannelId(SI(X=899.99, Z=399.99)) == S0 + 9 * 8 - 1
    for x, z in [(-1, 0), (1.7976931348623157e308, 0), (0, -1), (900, 400), (float("nan"), 0), (float("inf"), 0), (0, float("-inf"))]:
        with pytest.raises(SE):
            c.GetChannelId(SI(X=x, Z=z))


def test_kat_sphere_box_cone(chd):  # spatial_test.go:21-491
    c1 = _ctl(chd, 0, 0, 10, 10, 1, 1)
    assert S0 in c1.QueryChannelIds(_sphere(5, 5, 1))
    assert S0 in c1.QueryChannelIds(_sphere(5, 5, 100))
    assert S0 in c1.QueryChannelIds(_box(5, 5, 1, 1))
    assert S0 in c1.QueryChannelIds(_box(5, 5, 100, 100))
    assert S0 in c1.QueryChannelIds(_cone(5, 5, 1, 0, math.pi / 4, 1))
    c2 = _ctl(chd, -5, -5, 5, 5, 2, 2)
    assert len(c2.QueryChannelIds(_sphere(0, 0, 1))) == 4
    assert set(c2.QueryChannelIds(_sphere(4.9, 4.9, 1))) == {65539}
    assert len(c2.QueryChannelIds(_sphere(4.9, 4.9, 4.9))) == 1
    assert len(c2.QueryChannelIds(_sphere(4.9, 4.9, 10))) == 4
    assert len(c2.QueryChannelIds(_box(0, 0, 1, 1))) == 4
    assert set(c2.QueryChannelIds(_box(4.9, 4.9, 1, 1))) == {65539}
    assert len(c2.QueryChannelIds(_box(4.9, 4.9, 4.9, 4.9))) == 1
    assert set(c2.QueryChannelIds(_box(4.9, 4.9, 4.9, 10))) == {65539, 65537}
    c3 = _ctl(chd, -150, -150, 100, 100, 3, 3)
    assert len(c3.QueryChannelIds(_sphere(0, 0, 150))) == 9
    assert len(c3.QueryChannelIds(_sphere(0, 0, 99))) == 5
    assert len(c3.QueryChannelIds(_box(0, 0, 150, 150))) == 9
    assert len(c3.QueryChannelIds(_box(0, 0, 100, 100))) == 9
    g2 = _ctl(chd, 0, 0, 10, 10, 4, 1)
    assert S0 in g2.QueryChannelIds(_cone(0, 5, 1, 0, math.pi / 4, 1))
    assert len(g2.QueryChannelIds(_cone(0, 5, 1, 0, math.pi / 4, 25))) == 3
    assert len(g2.QueryChannelIds(_cone(0, 5, 1, 0, math.pi / 4, 100))) == 4
    assert len(g2.QueryChannelIds(_cone(0, 5, 0, 1, math.pi / 4, 100))) == 1
    g3 = _ctl(chd, 0, 0, 10, 10, 3, 3)
    assert set(g3.QueryChannelIds(_cone(5, 5, 1, 0, 0.1, 100))) == {65536, 65537, 65538}
    assert set(g3.QueryChannelIds(_cone(5, 5, 1, 0, math.pi / 4, 100))) == {65536, 65537, 65538, 65540, 65541, 65544}
    assert set(g3.QueryChannelIds(_cone(15, 15, -1, 0, math.pi / 4, 100))) == {65536, 65539, 65540, 65542}
    assert set(g3.QueryChannelIds(_cone(5, 15, 0, -1, math.pi / 4, 100))) == {65536, 65537, 65539}
    g4 = _ctl(chd, -2000, -500, 1000, 1000, 4, 1, 2, 1, 1)
    assert len(g4.QueryChannelIds(_cone(1250, 0, -0.087, 0.996, 0.5236, 30000))) == 1


def test_kat_adjacent_regions(chd, oracle):  # spatial_test.go:493-526 + GetRegions vs the oracle
    from tests._oracle import make_grid

    assert _ctl(chd, 0, 0, 10, 10, 1, 1, 1, 1, 1).GetAdjacentChannels(S0) == []
    assert len(_ctl(chd, -5, -5, 5, 5, 2, 2).GetAdjacentChannels(S0)) == 3
    c = _ctl(chd, -40, -60, 20, 40, 4, 3, 2, 3, 1)
    g = make_grid(-40, -60, 20, 40, 4, 3, 2, 3, 1)
    for cid in range(S0, S0 + 12):
        assert c.GetAdjacentChannels(cid) == oracle.adjacent(g, cid)
    regs = c.GetRegions()
    minx, minz, maxx, maxz, cid, srv = oracle.regions(g)
    for i, r in enumerate(regs):
        assert (r.Min.X, r.Min.Z, r.Max.X, r.Max.Z, r.ChannelId, r.ServerIndex) == (minx[i], minz[i], maxx[i], maxz[i], cid[i], srv[i])


# ----------------------------------------------------------------- randomized bit-exact parity of QueryChannelIds

GRIDS = [
    (-150, -150, 100, 100, 3, 3), (-5, -5, 5, 5, 2, 2), (0, 0, 10, 10, 4, 1), (-2000, -2000, 2000, 2000, 2, 2),
    (-15000, -15000, 2000, 2000, 15, 15), (-450, -200, 100, 50, 9, 8), (-12.5, 3.25, 7.3, 11.9, 13, 7), (0, 0, 33, 77, 2, 2),
]


def _random_queries(rng, g, n):
    offx, offz, w, h, cols, rows = g
    ww, wh = w * cols, h * rows
    C = __import__("channeld_b200.controller", fromlist=["x"])
    qs = []
    for _ in range(n):
        kind = rng.integers(0, 8)
        cx = offx + rng.uniform(-0.1, 1.1) * ww
        cz = offz + rng.uniform(-0.1, 1.1) * wh
        r = float(rng.choice([rng.uniform(0.01, 0.4) * min(w, h), rng.uniform(0.4, 3.0) * max(w, h), w * 0.5, h, 0.0, -1.0],
                             p=[0.4, 0.35, 0.1, 0.1, 0.03, 0.02]))
        q = C.SpatialInterestQuery()
        if kind in (0, 1, 2, 6):
            q.SphereAOI = C.SphereAOI(Center=C.SpatialInfo(X=cx, Z=cz), Radius=r)
        if kind in (3, 6, 7):
            q.BoxAOI = C.BoxAOI(Center=C.SpatialInfo(X=cx + rng.uniform(-1, 1) * w, Z=cz), Extent=C.SpatialInfo(
                X=abs(r) * rng.uniform(0.2, 1.5) if r > 0 else r, Z=rng.uniform(0.05, 2.5) * h))
        if kind in (4, 7):
            ang = rng.uniform(0, 2 * math.pi)
            q.ConeAOI = C.ConeAOI(Center=C.SpatialInfo(X=cx, Z=cz), Direction=C.SpatialInfo(X=math.cos(ang), Z=math.sin(ang)),
                                  Angle=float(rng.choice([0.1, math.pi / 4, 0.5236, rng.uniform(0, 3.2)])), Radius=abs(r) + 0.5 * w)
        if kind in (5, 6):
            k = int(rng.integers(1, 7))
            spots = [C.SpatialInfo(X=offx + rng.uniform(-0.05, 1.05) * ww, Z=offz + rng.uniform(-0.05, 1.05) * wh) for _ in range(k)]
            q.SpotsAOI = C.SpotsAOI(Spots=spots, Dists=[int(v) for v in rng.integers(0, 5, size=int(rng.integers(0, k + 1)))])
        qs.append(q)
    return qs


def _oracle_query(oracle, og, q):
    kw = {}
    if q.SpotsAOI is not None:
        kw["spots"] = [(s.X, s.Z) for s in q.SpotsAOI.Spots]
        kw["spot_dists"] = list(q.SpotsAOI.Dists)
    if q.BoxAOI is not None:
        kw["box"] = (q.BoxAOI.Center.X, q.BoxAOI.Center.Z, q.BoxAOI.Extent.X, q.BoxAOI.Extent.Z)
    if q.SphereAOI is not None:
        kw["sphere"] = (q.SphereAOI.Center.X, q.SphereAOI.Center.Z, q.SphereAOI.Radius)
    if q.ConeAOI is not None:
        c = q.ConeAOI
        kw["cone"] = (c.Center.X, c.Center.Z, c.Direction.X, c.Direction.Z, c.Angle, c.Radius)
    return oracle.query(og, **kw)


@pytest.mark.parametrize("gi", range(len(GRIDS)))
def test_random_query_parity(chd, oracle, gi):
    from tests._oracle import make_grid

    g = GRIDS[gi]
    rng = np.random.default_rng(1234 + gi)
    c = chd.controller.GpuStaticGrid2DSpatialController(max_entities=16, max_subscribers=2048, max_queries=2048, max_spots=1 << 15,
                                                        max_window_cells=1 << 22, max_pairs=1 << 20)
    c.LoadConfig(dict(WorldOffsetX=g[0], WorldOffsetZ=g[1], GridWidth=g[2], GridHeight=g[3], GridCols=g[4], GridRows=g[5],
                      ServerCols=1, ServerRows=1))
    og = make_grid(*g)
    qs = _random_queries(rng, g, 1500)
    got = c.QueryChannelIdsBatch(qs)
    n_err = 0
    for q, res in zip(qs, got):
        want, st = _oracle_query(oracle, og, q)
        if st != 0:
            assert isinstance(res, chd.controller.SpatialError), (q, st)
            n_err += 1
        else:
            assert res == want, (q, res, want)
    assert 0 < n_err < len(qs)


def test_cell_of_parity_edges(chd, oracle):
    from tests._oracle import make_grid

    g = (-450, -200, 100, 50, 9, 8)
    c = _ctl(chd, *g)
    og = make_grid(*g)
    rng = np.random.default_rng(5)
    x = rng.uniform(-600, 600, 20000)
    z = rng.uniform(-300, 300, 20000)
    # exact cell boundaries and neighbours one ulp either side
    bx = -450 + 100.0 * np.arange(-1, 11)
    bz = -200 + 50.0 * np.arange(-1, 10)
    ex = np.concatenate([bx, np.nextafter(bx, -np.inf), np.nextafter(bx, np.inf), [np.nan, np.inf, -np.inf, 1e308, -1e308, 0.0, -0.0]])
    ez = np.concatenate([bz, np.nextafter(bz, -np.inf), np.nextafter(bz, np.inf)])
    xs = np.concatenate([x, np.repeat(ex, len(ez))])
    zs = np.concatenate([z, np.tile(ez, len(ex))])
    np.testing.assert_array_equal(c.GetChannelIds(xs, zs), oracle.cell_of(og, xs, zs))


# ----------------------------------------------------------------- build + full tick on BASELINE config #1

def _oracle_grid(wc):
    from tests._oracle import make_grid

    return make_grid(wc.offx, wc.offz, wc.w, wc.h, wc.cols, wc.rows, wc.server_cols, wc.server_rows)


@pytest.mark.parametrize("radius", [50.0, 500.0, 2500.0])
def test_tick_config1_full_parity(chd, oracle, radius):
    """config #1: spatial_static_2x2, 1K entities / 256 subscribers: pairs + visible lists bit-identical."""
    wc = chd.synth.CONFIGS["2x2"]
    ex, ez = chd.synth.entities(wc)
    conn, cx, cz, r = chd.synth.subscribers(wc, ex, ez, radius)
    want = oracle.sphere_tick(_oracle_grid(wc), ex, ez, cx, cz, r)
    e = chd.engine.Engine(wc.cfg(), wc.n_entities, wc.n_subscribers, max_visible=1 << 20)
    e.set_entities(ex, ez)
    e.set_subscribers(conn)
    batch, keep = chd.engine.make_batch(len(cx), sub=np.arange(len(cx), dtype=np.uint32), sphere=(cx, cz, r))
    s = e.tick(batch, 0, chd.capi.TICK_BUILD | chd.capi.TICK_EMIT)
    assert s.n_pairs == len(want["pair_cell"]) and s.n_visible == len(want["vis_entity"])
    assert s.n_query_errors == int((want["status"] != 0).sum())
    pairs = e.get_pairs()
    np.testing.assert_array_equal(pairs["off"].astype(np.uint64), want["pair_off"])
    np.testing.assert_array_equal(pairs["channel"], want["pair_cell"])
    np.testing.assert_array_equal(pairs["dist"], want["pair_dist"])
    np.testing.assert_array_equal(pairs["interval"], [oracle.damping(int(d), 20) for d in want["pair_dist"]])
    voff, vis = e.get_visible()
    np.testing.assert_array_equal(voff, want["vis_off"])
    np.testing.assert_array_equal(vis, want["vis_entity"])
    np.testing.assert_array_equal(e.get_query_status(len(cx)), want["status"])
    # cell CSR against a stable CPU sort of the oracle's cell ids
    cs, se = e.get_cells()
    ids = oracle.cell_of(_oracle_grid(wc), ex, ez)
    valid = np.nonzero(ids)[0]
    order = valid[np.argsort(ids[valid], kind="stable")]
    np.testing.assert_array_equal(se, order.astype(np.uint32))
    np.testing.assert_array_equal(cs, np.concatenate([[0], np.cumsum(np.bincount(ids[valid] - S0, minlength=wc.cells))]))
    assert s.n_entities_in_world == len(valid)


@pytest.mark.parametrize("name,n_ent,n_sub", [("benchmark", 200_000, 20_000), ("10m", 300_000, 30_000), ("handover", 400_000, 4_000)])
def test_tick_scaled_configs_parity(chd, oracle, name, n_ent, n_sub):
    """The grids of configs #2/#3/#5 (1- and 2-pass radix build, 225 / 4096 / 65536 cells) at sizes the oracle
    finishes in seconds: pairs + visible lists bit-identical."""
    wc = chd.synth.scaled(chd.synth.CONFIGS[name], n_ent, n_sub)
    ex, ez = chd.synth.entities(wc)
    # push some entities out of the world / onto the max edge
    ex[::1013] = wc.offx + wc.w * wc.cols
    ez[::2027] = wc.offz - 1.0
    conn, cx, cz, r = chd.synth.subscribers(wc, ex, ez)
    want = oracle.sphere_tick(_oracle_grid(wc), ex, ez, cx, cz, r)
    e = chd.engine.Engine(wc.cfg(), n_ent, n_sub, max_visible=int(len(want["vis_entity"]) + 4096))
    e.set_entities(ex, ez)
    e.set_subscribers(conn)
    # "10m" uses the identity batch (sub = NULL: query i <-> subscriber slot i), the others an explicit slot table
    batch, keep = chd.engine.make_batch(n_sub, sub=None if name == "10m" else np.arange(n_sub, dtype=np.uint32), sphere=(cx, cz, r))
    s = e.tick(batch, 0, chd.capi.TICK_BUILD | chd.capi.TICK_EMIT)
    assert s.n_pairs == len(want["pair_cell"]) and s.n_visible == len(want["vis_entity"])
    pairs = e.get_pairs()
    np.testing.assert_array_equal(pairs["off"].astype(np.uint64), want["pair_off"])
    np.testing.assert_array_equal(pairs["channel"], want["pair_cell"])
    np.testing.assert_array_equal(pairs["dist"], want["pair_dist"])
    voff, vis = e.get_visible()
    np.testing.assert_array_equal(voff, want["vis_off"])
    np.testing.assert_array_equal(vis, want["vis_entity"])
    np.testing.assert_array_equal(e.get_query_status(n_sub), want["status"])


def test_visible_overflow_reported(chd):
    wc = chd.synth.CONFIGS["2x2"]
    ex, ez = chd.synth.entities(wc)
    conn, cx, cz, r = chd.synth.subscribers(wc, ex, ez, 2500.0)
    e = chd.engine.Engine(wc.cfg(), wc.n_entities, wc.n_subscribers, max_visible=1000)
    e.set_entities(ex, ez)
    e.set_subscribers(conn)
    batch, keep = chd.engine.make_batch(len(cx), sub=np.arange(len(cx), dtype=np.uint32), sphere=(cx, cz, r))
    with pytest.raises(chd.capi.ChdError) as ei:
        e.tick(batch, 0, chd.capi.TICK_BUILD | chd.capi.TICK_EMIT)
    assert ei.value.status == chd.capi.ERR_CAPACITY


# ----------------------------------------------------------------- interest diff + fan-out over several ticks

def test_interest_diff_and_fanout_parity(chd, oracle):
    """Moving subscribers on a 6x5 grid over 12 ticks: per tick the sub/unsub/kept sets match
    oracle.interest_diff, and every fan-out decision matches the literal emulation of Channel.tickData
    (one oracle channel per cell, fed the same subscriptions and update rings)."""
    g = (-300.0, -250.0, 100.0, 100.0, 6, 5)
    from tests._oracle import make_grid

    og = make_grid(*g)
    rng = np.random.default_rng(99)
    S, N = 60, 500
    cfg = chd.engine.grid_cfg(*g)
    e = chd.engine.Engine(cfg, N, S, max_visible=1 << 20)
    conn = np.arange(101, 101 + S, dtype=np.uint32)
    e.set_subscribers(conn)
    ex, ez = rng.uniform(-300, 300, N), rng.uniform(-250, 250, N)
    e.set_entities(ex, ez)
    e.build()
    cells = g[4] * g[5]
    chans = [oracle.channel() for _ in range(cells)]
    rings = [[] for _ in range(cells)]  # (arrival, sender, index)
    msg_index = np.zeros(cells, np.uint64)
    cx, cz = rng.uniform(-320, 320, S), rng.uniform(-270, 270, S)  # a few start outside the world
    rad = rng.choice([30.0, 60.0, 120.0, 260.0], S)
    subs_now = [dict() for _ in range(S)]  # channel id -> dist, the oracle-side spatialSubscriptions
    t = 0
    tick_ns = 33 * MS
    total_due = total_classes = total_shared = 0
    for tick in range(12):
        t += tick_ns if tick % 4 else 70 * MS  # irregular ticks exercise multi-step catch-up
        cx += rng.uniform(-45, 45, S)
        cz += rng.uniform(-45, 45, S)
        moving = rng.random(S) < 0.8  # the others send no UPDATE_SPATIAL_INTEREST this tick
        qi = np.nonzero(moving)[0].astype(np.uint32)
        batch, keep = chd.engine.make_batch(len(qi), sub=qi, sphere=(cx[qi], cz[qi], rad[qi]))
        e.update_interest(batch, t)
        s = e.summary()
        (new_s, new_c), (un_s, un_c) = e.get_diff(s.n_sub_new, s.n_unsub)
        want_new, want_un, n_kept = set(), set(), 0
        for j in qi:
            res, st = oracle.query(og, sphere=(cx[j], cz[j], rad[j]))
            if st != 0:
                continue
            un, sn, kp = oracle.interest_diff(list(subs_now[j].keys()), list(res.keys()))
            for c in un:
                want_un.add((int(j), int(c)))
                chans[c - S0].unsubscribe(int(conn[j]))
                del subs_now[j][int(c)]
            for c in list(sn) + list(kp):
                iv = oracle.damping(res[int(c)], 20)
                chans[c - S0].subscribe(int(conn[j]), t, iv, 0, True, False)
                subs_now[j][int(c)] = res[int(c)]
            want_new |= {(int(j), int(c)) for c in sn}
            n_kept += len(kp)
        assert set(zip(new_s.tolist(), new_c.tolist())) == want_new
        assert set(zip(un_s.tolist(), un_c.tolist())) == want_un
        assert (s.n_sub_new, s.n_unsub, s.n_kept) == (len(want_new), len(want_un), n_kept)
        pairs = e.get_pairs()
        for j in range(S):
            sl = slice(pairs["off"][j], pairs["off"][j + 1])
            assert dict(zip(pairs["channel"][sl].tolist(), pairs["dist"][sl].tolist())) == subs_now[j]
        # updates arrive (some sent by subscribers themselves -> SkipSelfUpdateFanOut)
        for _ in range(int(rng.integers(5, 40))):
            c = int(rng.integers(0, cells))
            arrival = t - int(rng.integers(0, 80)) * MS  # not time-sorted on purpose (data_test.go:70-94)
            sender = int(rng.choice(conn)) if rng.random() < 0.5 else 7
            msg_index[c] += 1
            rings[c].append((arrival, sender, int(msg_index[c])))
            chans[c].on_update(arrival, sender)
        ring_off = np.concatenate([[0], np.cumsum([len(r) for r in rings])]).astype(np.uint32)
        flat = [x for r in rings for x in r]
        e.set_rings(ring_off, np.array([f[0] for f in flat], np.int64), np.array([f[1] for f in flat], np.uint32),
                    np.array([f[2] for f in flat], np.uint64), msg_index)
        e.fanout_tick(t)
        s = e.summary()
        due = e.get_due(s.n_due)
        want, want_ex = [], {}
        for c in range(cells):
            for d in chans[c].tick_data_ex(t):
                want.append((d["conn"], S0 + c, d["kind"], d["n"], d["first"], d["last"], d["hash"], d["last_index"], d["window_hi"]))
                want_ex[(d["conn"], S0 + c, d["kind"], d["window_hi"])] = d
        got = [(int(conn[d["sub"]]), int(d["channel_id"]), int(d["kind"]), int(d["n_selected"]), int(d["first_sel"]), int(d["last_sel"]),
                int(d["sel_hash"]), int(d["last_message_index"]), int(d["window_hi"])) for d in due]
        assert sorted(got) == sorted(want)
        total_due += len(got)
        # window classes (chd_due_classes): decisions grouped by payload identity
        cls_of, cls_rep, cls_cnt = e.due_classes(s.n_due)
        assert len(want_ex) == len(want)
        exact, doc = [], []
        for g_ in got:
            w = want_ex[(g_[0], g_[1], g_[2], g_[8])]
            if g_[2] == 0:
                exact.append((g_[1], 0)); doc.append((g_[1], 0))
            else:
                exact.append((g_[1], 1, w["selected"]))  # the ring entries actually merged (oracle emulation)
                doc.append((g_[1], 1, w["window_lo"], w["window_hi"], g_[0] if w["self_skipped"] else 0))
        members = {}
        for i, k in enumerate(cls_of.tolist()):
            members.setdefault(k, []).append(i)
        assert sorted(members) == list(range(len(cls_rep)))
        for k, idx in members.items():
            assert len({exact[i] for i in idx}) == 1, "a class mixes different payloads"
            assert len({doc[i] for i in idx}) == 1
            assert cls_rep[k] == min(idx) and cls_cnt[k] == len(idx)
        assert len({doc[i] for i in range(len(got))}) == len(cls_rep)  # no identity is split over two classes
        assert cls_rep.tolist() == sorted(cls_rep.tolist())
        total_classes += len(cls_rep)
        total_shared += len(got) - len(cls_rep)
        # committed state matches the oracle's fanOutConnection
        pairs = e.get_pairs()
        for j in range(S):
            for p in range(pairs["off"][j], pairs["off"][j + 1]):
                last, had, idx = chans[int(pairs["channel"][p]) - S0].state(int(conn[j]))
                assert (int(pairs["last"][p]), bool(pairs["flags"][p] & 1), int(pairs["last_index"][p])) == (last, had, idx)
    assert total_due > 200 and 0 < total_classes < total_due and total_shared > 50


def test_fanout_kat_through_engine(chd):
    """data_test.go:98-166 (F0, F7, F2, F8=U1+U2, F3) replayed through chd_fanout_tick on a 1x1 grid."""
    cfg = chd.engine.grid_cfg(0, 0, 10, 10, 1, 1)
    e = chd.engine.Engine(cfg, 4, 4, default_fanout_interval_ms=50)
    e.set_entities(np.array([5.0]), np.array([5.0]))
    e.build()
    e.set_subscribers(np.array([1, 2, 3], np.uint32))  # slots: c0=server(sender), c1, c2

    def interest(slots, t):
        # dist 0 -> 20 ms would apply; use a cone-free trick: SpotsAOI with explicit dists selects the interval:
        # dist 1 -> 50 ms (c1), dist 2 -> 100 ms (c2)   (message_spatial.go:16-38)
        n = len(slots)
        off = np.arange(n + 1, dtype=np.uint32)
        b, keep = chd.engine.make_batch(n, sub=np.array([s for s, _ in slots], np.uint32), kind=np.full(n, chd.capi.AOI_SPOTS, np.uint8),
                                        spots=(off, np.ones(n, np.uint32), np.full(n, 5.0), np.full(n, 5.0),
                                               np.array([d for _, d in slots], np.uint32)))
        e.update_interest(b, t)

    def tick(t, ring):
        off = np.array([0, len(ring)], np.uint32)
        e.set_rings(off, np.array([r[0] for r in ring], np.int64), np.array([r[1] for r in ring], np.uint32),
                    np.array([r[2] for r in ring], np.uint64), np.array([len(ring)], np.uint64))
        e.fanout_tick(t)
        s = e.summary()
        return e.get_due(s.n_due)

    t0 = 100 * MS
    interest([(1, 1)], 0)  # c1 subscribes at ~0 with 50 ms
    due = tick(t0, [])
    assert [(int(d["sub"]), int(d["kind"])) for d in due] == [(1, 0)]  # F0 = whole data
    interest([(2, 2)], 0)  # c2 subscribes with 100 ms (channel time ~0 in the reference test)
    due = tick(t0 + 50 * MS, [])
    assert [(int(d["sub"]), int(d["kind"])) for d in due] == [(2, 0)]  # F1 nothing, F7 whole data
    ring = [(t0 + 60 * MS, 1, 1)]  # U1 from c0 (conn id 1)
    due = tick(t0 + 100 * MS, ring)
    assert [(int(d["sub"]), int(d["kind"]), int(d["n_selected"]), int(d["sel_hash"])) for d in due] == [(1, 1, 1, 1)]  # F2 = U1
    ring.append((t0 + 120 * MS, 1, 2))  # U2
    due = tick(t0 + 150 * MS, ring)
    assert sorted((int(d["sub"]), int(d["n_selected"]), int(d["sel_hash"])) for d in due) == [(1, 1, 2), (2, 2, 3)]  # F3=U2, F8=U1+U2


def test_handover_detection(chd, oracle):
    wc = chd.synth.scaled(chd.synth.CONFIGS["handover"], 50_000, 16)
    ex, ez = chd.synth.entities(wc)
    og = _oracle_grid(wc)
    c = chd.controller.GpuStaticGrid2DSpatialController(max_entities=50_000, max_subscribers=16)
    c.LoadConfig(dict(WorldOffsetX=wc.offx, WorldOffsetZ=wc.offz, GridWidth=wc.w, GridHeight=wc.h, GridCols=wc.cols, GridRows=wc.rows,
                      ServerCols=1, ServerRows=1))
    ent, src, dst = c.NotifyBatch(ex, ez)
    assert len(ent) == 0
    nx, nz = chd.synth.move_entities(wc, ex, ez, 1, 60.0)
    nx[:5] = wc.offx - 10.0  # leave the world: the reference logs "failed to calculate dstChannelId"
    ent, src, dst = c.NotifyBatch(nx, nz)
    old, new = oracle.cell_of(og, ex, ez), oracle.cell_of(og, nx, nz)
    moved = np.nonzero(old != new)[0]
    order = np.argsort(ent)
    np.testing.assert_array_equal(ent[order], moved.astype(np.uint32))
    np.testing.assert_array_equal(src[order], old[moved])
    np.testing.assert_array_equal(dst[order], new[moved])
    assert len(moved) > 1000


def test_graph_replay_matches_direct_and_oracle(chd, oracle):
    """Six full ticks with moving entities: the CUDA-graph replay path (stable shapes) must give the same pairs,
    visible lists, diff counts, handover lists and fan-out decisions as direct launches, and match the oracle."""
    wc = chd.synth.scaled(chd.synth.CONFIGS["benchmark"], 30_000, 3_000)
    og = _oracle_grid(wc)
    results = {}
    for use_graphs in (True, False):
        e = chd.engine.Engine(wc.cfg(), wc.n_entities, wc.n_subscribers, max_visible=1 << 22)
        e.enable_graphs(use_graphs)
        ex, ez = chd.synth.entities(wc)
        conn, _, _, _ = chd.synth.subscribers(wc, ex, ez)
        e.set_subscribers(conn)
        ring_state, out = None, []
        for tick in range(6):
            t = (tick + 1) * 33_000_000
            ex, ez = chd.synth.move_entities(wc, ex, ez, tick, 400.0)
            _, cx, cz, r = chd.synth.subscribers(wc, ex, ez)
            e.set_entities(ex, ez)
            batch, keep = chd.engine.make_batch(len(cx), sub=np.arange(len(cx), dtype=np.uint32), sphere=(cx, cz, r))
            ring_state, off, arr, snd, idx, cmi = chd.synth.update_rings(wc, tick, t, 33_000_000, 4, len(conn), ring_len=16, state=ring_state)
            e.set_rings(off, arr, snd, idx, cmi)
            if use_graphs and tick % 2:
                # early-start path: interest + fan-out begin on the second stream before the positions are uploaded
                e.begin_interest(batch, t, with_fanout=True)
                e.set_entities(ex, ez)
                s = e.tick(None, t, chd.capi.TICK_ALL)
            else:
                s = e.tick(batch, t, chd.capi.TICK_ALL)
            pairs = e.get_pairs(s.n_pairs)
            voff, vis = e.get_visible()
            due = e.get_due(s.n_due)
            due = due[np.lexsort((due["window_hi"], due["channel_id"], due["sub"]))]  # the due list is a set: canonical order
            ho = e.get_handover(s.n_handover)
            order = np.argsort(ho[0])
            out.append((s.as_dict(), pairs, voff, vis, due, tuple(a[order] for a in ho)))
            if use_graphs:
                want = oracle.sphere_tick(og, ex, ez, cx, cz, r)
                np.testing.assert_array_equal(pairs["channel"], want["pair_cell"])
                np.testing.assert_array_equal(pairs["dist"], want["pair_dist"])
                np.testing.assert_array_equal(voff, want["vis_off"])
                np.testing.assert_array_equal(vis, want["vis_entity"])
        results[use_graphs] = out
        if use_graphs:
            assert e.graph_launch_count() >= 8, e.graph_launch_count()
        else:
            assert e.graph_launch_count() == 0
    for a, b in zip(results[True], results[False]):
        assert a[0] == b[0]
        for k in a[1]:
            np.testing.assert_array_equal(a[1][k], b[1][k])
        np.testing.assert_array_equal(a[2], b[2])
        np.testing.assert_array_equal(a[3], b[3])
        np.testing.assert_array_equal(a[4], b[4])
        for x, y in zip(a[5], b[5]):
            np.testing.assert_array_equal(x, y)
    assert sum(r[0]["n_due"] for r in results[True]) > 1000 and sum(r[0]["n_handover"] for r in results[True]) > 100


def test_tick_forms_match_step_by_step(chd):
    """Every way of enqueueing a tick (one stream or two, the interest / fan-out chain started by chd_tick or early by
    chd_begin_interest with or without the fan-out, the fan-out on the main stream after the join, the early read-back)
    gives the summary, pairs, visible lists, interest diff, due list and handover list of the four stages called one by one."""
    import ctypes as C

    wc = chd.synth.scaled(chd.synth.CONFIGS["benchmark"], 30_000, 3_000)
    A, B, E, F = chd.capi.TICK_ALL, chd.capi.TICK_BUILD, chd.capi.TICK_EMIT, chd.capi.TICK_FANOUT

    def step(e, batch, t):
        e.build()
        e.update_interest(batch, t)
        e.emit_visible()
        e.fanout_tick(t)
        return e.summary()

    def early(e, batch, t):
        e.tick(batch, t, A | chd.capi.TICK_EARLY_RESULTS, want_summary=False)
        s = chd.capi.TickSummary()
        e._ck(e.L.chd_fetch_results(e.h, C.byref(chd.capi.ResultBuffers()), C.byref(s)))
        return s

    def begin(with_fanout):
        def run(e, batch, t):
            e.begin_interest(batch, t, with_fanout=with_fanout)
            return e.tick(None, t, A)
        return run

    def build_emit_then_fanout(e, batch, t):
        e.tick(batch, t, B | E, want_summary=False)
        e.fanout_tick(t)
        return e.summary()

    forms = {"step": step, "tick": lambda e, batch, t: e.tick(batch, t, A), "early_results": early,
             "begin_with_fanout": begin(True), "begin_without_fanout": begin(False), "build_emit_then_fanout": build_emit_then_fanout}
    canon = lambda u, v: np.sort(u.astype(np.uint64) << np.uint64(32) | v.astype(np.uint64))  # noqa: E731
    results = {}
    for name, run in forms.items():
        e = chd.engine.Engine(wc.cfg(), wc.n_entities, wc.n_subscribers, max_visible=1 << 22)
        ex, ez = chd.synth.entities(wc)
        conn, _, _, _ = chd.synth.subscribers(wc, ex, ez)
        e.set_subscribers(conn)
        ring_state, out = None, []
        for tick in range(4):
            t = (tick + 1) * 33_000_000
            ex, ez = chd.synth.move_entities(wc, ex, ez, tick, 400.0)
            _, cx, cz, r = chd.synth.subscribers(wc, ex, ez)
            ring_state, off, arr, snd, idx, cmi = chd.synth.update_rings(wc, tick, t, 33_000_000, 4, len(conn), ring_len=16, state=ring_state)
            e.set_rings(off, arr, snd, idx, cmi)
            e.set_entities(ex, ez)
            batch, keep = chd.engine.make_batch(len(cx), sub=np.arange(len(cx), dtype=np.uint32), sphere=(cx, cz, r))
            s = run(e, batch, t)
            pairs = e.get_pairs(s.n_pairs)
            voff, vis = e.get_visible()
            (ns, nc), (us, uc) = e.get_diff(s.n_sub_new, s.n_unsub)
            due = e.get_due(s.n_due)
            due = due[np.lexsort((due["window_hi"], due["channel_id"], due["sub"]))]
            ho = np.stack(e.get_handover(s.n_handover), 1)
            ho = ho[np.lexsort((ho[:, 2], ho[:, 1], ho[:, 0]))]
            out.append(dict(s=s.as_dict(), pairs=pairs, voff=voff, vis=vis, new=canon(ns, nc), unsub=canon(us, uc), due=due, ho=ho))
        e.close()
        results[name] = out
    want = results.pop("step")
    for k in ("n_due", "n_handover", "n_sub_new", "n_unsub"):  # every compared list is non-empty in some tick
        assert sum(w["s"][k] for w in want) > 0, k
    for name, got in results.items():
        for tick, (g, w) in enumerate(zip(got, want)):
            assert g["s"] == w["s"], (name, tick)
            for k in w["pairs"]:
                np.testing.assert_array_equal(g["pairs"][k], w["pairs"][k], err_msg=f"{name} tick {tick} pairs {k}")
            for k in ("voff", "vis", "new", "unsub", "due", "ho"):
                np.testing.assert_array_equal(g[k], w[k], err_msg=f"{name} tick {tick} {k}")


@pytest.mark.parametrize("early", [False, True])
def test_fetch_results_matches_getters(chd, early):
    """chd_fetch_results (one call) returns exactly what the individual getters return, also when the read-back runs
    on its own stream while the expanded-list kernel is still in flight (CHD_TICK_EARLY_RESULTS)."""
    import ctypes as C

    wc = chd.synth.scaled(chd.synth.CONFIGS["benchmark"], 20_000, 2_000)
    e = chd.engine.Engine(wc.cfg(), wc.n_entities, wc.n_subscribers, max_visible=1 << 22)
    ex, ez = chd.synth.entities(wc)
    conn, cx, cz, r = chd.synth.subscribers(wc, ex, ez)
    cx[:3] = wc.offx - 5.0  # a few failing queries
    e.set_subscribers(conn)
    ring_state = None
    for tick in range(3):
        t = (tick + 1) * 33_000_000
        ex, ez = chd.synth.move_entities(wc, ex, ez, tick, 500.0)
        e.set_entities(ex, ez)
        cq = cx.copy()
        cq[3:] += 300.0 * tick  # the first three stay outside the world
        batch, keep = chd.engine.make_batch(len(cx), sub=np.arange(len(cx), dtype=np.uint32), sphere=(cq, cz, r))
        ring_state, off, arr, snd, idx, cmi = chd.synth.update_rings(wc, tick, t, 33_000_000, 4, len(conn), ring_len=16, state=ring_state)
        e.set_rings(off, arr, snd, idx, cmi)
        e.tick(batch, t, chd.capi.TICK_ALL | (chd.capi.TICK_EARLY_RESULTS if early else 0), want_summary=False)
        S, cap = len(conn), 1 << 16
        bufs = {k: np.zeros(cap, np.uint32) for k in ("ch", "dist", "iv", "ns", "nc", "us", "uc", "he", "hs", "hd", "st", "se")}
        poff, voff = np.zeros(S + 1, np.uint32), np.zeros(S + 1, np.uint64)
        due = np.zeros(cap, chd.capi.DUE_DTYPE)
        vis = np.zeros(1 << 22, np.uint32)
        cs = np.zeros(wc.cells + 1, np.uint32)
        rb = chd.capi.ResultBuffers()
        P = chd.capi.ptr
        rb.pair_off, rb.pair_channel, rb.pair_dist, rb.pair_interval_ms, rb.pair_cap = P(poff), P(bufs["ch"]), P(bufs["dist"]), P(bufs["iv"]), cap
        rb.new_sub, rb.new_channel, rb.unsub_sub, rb.unsub_channel, rb.diff_cap = P(bufs["ns"]), P(bufs["nc"]), P(bufs["us"]), P(bufs["uc"]), cap
        rb.due, rb.due_cap = P(due), cap
        rb.handover_entity, rb.handover_src, rb.handover_dst, rb.handover_cap = P(bufs["he"]), P(bufs["hs"]), P(bufs["hd"]), cap
        rb.query_status, rb.status_cap = P(bufs["st"]), cap
        rb.vis_off, rb.vis_entity, rb.vis_cap = P(voff), P(vis), len(vis)
        rb.cell_start, rb.sorted_entity, rb.entity_cap = P(cs), P(bufs["se"]), cap
        s = chd.capi.TickSummary()
        assert e.L.chd_fetch_results(e.h, C.byref(rb), C.byref(s)) == 0
        pairs = e.get_pairs(s.n_pairs)
        np.testing.assert_array_equal(poff, pairs["off"])
        for k, name in (("ch", "channel"), ("dist", "dist"), ("iv", "interval")):
            np.testing.assert_array_equal(bufs[k][:s.n_pairs], pairs[name])
        (a, b), (c, d) = e.get_diff(s.n_sub_new, s.n_unsub)
        np.testing.assert_array_equal(bufs["ns"][:s.n_sub_new], a); np.testing.assert_array_equal(bufs["nc"][:s.n_sub_new], b)
        np.testing.assert_array_equal(bufs["us"][:s.n_unsub], c); np.testing.assert_array_equal(bufs["uc"][:s.n_unsub], d)
        np.testing.assert_array_equal(due[:s.n_due], e.get_due(s.n_due))
        h = e.get_handover(s.n_handover)
        for k, arr_ in zip(("he", "hs", "hd"), h):
            np.testing.assert_array_equal(bufs[k][:s.n_handover], arr_)
        np.testing.assert_array_equal(bufs["st"][:len(cx)], e.get_query_status(len(cx)))
        v0, v1 = e.get_visible()
        np.testing.assert_array_equal(voff, v0); np.testing.assert_array_equal(vis[:s.n_visible], v1)
        c0, c1 = e.get_cells()
        np.testing.assert_array_equal(cs, c0); np.testing.assert_array_equal(bufs["se"][:s.n_entities_in_world], c1)
        assert s.n_query_errors == int((bufs["st"][:len(cx)] != 0).sum()) >= 3 and (bufs["st"][:3] == chd.capi.Q_ERR_OUT_OF_WORLD).all()
    # too small a capacity is an error, never a silent truncation
    rb.pair_cap = 1
    assert e.L.chd_fetch_results(e.h, C.byref(rb), C.byref(s)) == chd.capi.ERR_CAPACITY


def test_async_fetch_matches_getters_while_the_next_tick_runs(chd):
    """chd_fetch_results_async / chd_fetch_wait: tick k+1 is enqueued (and overwrites the engine's result arrays) BEFORE the host
    waits for tick k's results; what arrives in the pinned buffers equals what a second engine's getters return for tick k.  Also:
    a third outstanding fetch is refused."""
    import ctypes as C

    import torch

    wc = chd.synth.scaled(chd.synth.CONFIGS["benchmark"], 50_000, 4_000)
    ex, ez = chd.synth.entities(wc)
    conn, _, _, _ = chd.synth.subscribers(wc, ex, ez)
    frames, ring_state = [], None
    for tick in range(6):
        t = (tick + 1) * 33_000_000
        ex, ez = chd.synth.move_entities(wc, ex, ez, tick, 400.0)
        _, cx, cz, r = chd.synth.subscribers(wc, ex, ez)
        ring_state, off, arr, snd, idx, cmi = chd.synth.update_rings(wc, tick, t, 33_000_000, 4, len(conn), ring_len=16, state=ring_state)
        frames.append(dict(t=t, x=ex.copy(), z=ez.copy(), q=(cx, cz, r), rings=(off, arr, snd, idx, cmi)))
    S, cap = len(conn), 1 << 17

    def pin(n, dt):
        t_ = torch.zeros(n, dtype=dt).pin_memory()
        return t_, t_.numpy()

    def result_set():
        k = {n_: pin(cap, torch.int32) for n_ in ("ch", "dist", "iv", "ns", "nc", "us", "uc", "he", "hs", "hd", "st", "se")}
        k["off"], k["voff"], k["cs"] = pin(S + 1, torch.int32), pin(S + 1, torch.int64), pin(wc.cells + 1, torch.int32)
        k["due"], k["hdr"] = pin(cap * 12, torch.int32), pin(64, torch.int32)
        rb = chd.capi.ResultBuffers()
        P = lambda n_: chd.capi.ptr(k[n_][0])  # noqa: E731
        rb.pair_off, rb.pair_channel, rb.pair_dist, rb.pair_interval_ms, rb.pair_cap = P("off"), P("ch"), P("dist"), P("iv"), cap
        rb.new_sub, rb.new_channel, rb.unsub_sub, rb.unsub_channel, rb.diff_cap = P("ns"), P("nc"), P("us"), P("uc"), cap
        rb.due, rb.due_cap = P("due"), cap
        rb.handover_entity, rb.handover_src, rb.handover_dst, rb.handover_cap = P("he"), P("hs"), P("hd"), cap
        rb.query_status, rb.status_cap = P("st"), cap
        rb.vis_off, rb.vis_entity, rb.vis_cap = P("voff"), None, 0
        rb.cell_start, rb.sorted_entity, rb.entity_cap = P("cs"), P("se"), cap
        return rb, k

    # the plain engine: one synchronous tick at a time, getters
    e1 = chd.engine.Engine(wc.cfg(), wc.n_entities, wc.n_subscribers, max_visible=1 << 24)
    e1.set_subscribers(conn)
    want = []
    for f in frames:
        e1.set_rings(*f["rings"])
        e1.set_entities(f["x"], f["z"])
        batch, keep = chd.engine.make_batch(S, sub=None, sphere=f["q"])
        s = e1.tick(batch, f["t"], chd.capi.TICK_ALL)
        voff, _ = e1.get_visible()
        cs, se = e1.get_cells()
        want.append(dict(s=s.as_dict(), pairs=e1.get_pairs(s.n_pairs), diff=e1.get_diff(s.n_sub_new, s.n_unsub), due=e1.get_due(s.n_due),
                         ho=e1.get_handover(s.n_handover), st=e1.get_query_status(S), voff=voff, cs=cs, se=se))
    e1.close()

    e = chd.engine.Engine(wc.cfg(), wc.n_entities, wc.n_subscribers, max_visible=1 << 24)
    e.set_subscribers(conn)
    sets = [result_set(), result_set()]
    ck = e._ck

    def prefetch(f):
        batch, keep = chd.engine.make_batch(S, sub=None, sphere=f["q"])
        e.prefetch_rings(*f["rings"])
        e.prefetch_queries(batch, keep)
        e.prefetch_entities(f["x"], f["z"])

    def enqueue(i):
        e.adopt_prefetched()
        e.begin_interest(None, frames[i]["t"])
        ck(e.L.chd_tick(e.h, None, frames[i]["t"], chd.capi.TICK_ALL, None))
        if i + 1 < len(frames):
            prefetch(frames[i + 1])
        rb, k = sets[i % 2]
        ck(e.L.chd_fetch_results_async(e.h, C.byref(rb), chd.capi.ptr(k["hdr"][0])))

    def check(i, s):
        w, k = want[i], sets[i % 2][1]
        assert s.as_dict() == w["s"], i
        n = s.n_pairs
        np.testing.assert_array_equal(k["off"][1].view(np.uint32), w["pairs"]["off"])
        for a, b in (("ch", "channel"), ("dist", "dist"), ("iv", "interval")):
            np.testing.assert_array_equal(k[a][1][:n].view(np.uint32), w["pairs"][b])
        (a, b), (c, d) = w["diff"]
        # (the sub / unsub lists are appended block by block: sets of (subscriber, channel), compared in a canonical order)
        canon = lambda u, v: np.sort(u.astype(np.uint64) << np.uint64(32) | v.astype(np.uint64))  # noqa: E731
        np.testing.assert_array_equal(canon(k["ns"][1][:s.n_sub_new].view(np.uint32), k["nc"][1][:s.n_sub_new].view(np.uint32)), canon(a, b))
        np.testing.assert_array_equal(canon(k["us"][1][:s.n_unsub].view(np.uint32), k["uc"][1][:s.n_unsub].view(np.uint32)), canon(c, d))
        got_due = k["due"][1][:s.n_due * 12].view(chd.capi.DUE_DTYPE)
        key = lambda d_: d_[np.lexsort((d_["window_hi"], d_["channel_id"], d_["sub"]))]  # noqa: E731
        np.testing.assert_array_equal(key(got_due), key(w["due"]))
        ho_g = np.stack([k[a][1][:s.n_handover].view(np.uint32) for a in ("he", "hs", "hd")], 1)
        ho_w = np.stack(w["ho"], 1)
        srt = lambda h: h[np.lexsort((h[:, 2], h[:, 1], h[:, 0]))]  # noqa: E731
        np.testing.assert_array_equal(srt(ho_g), srt(ho_w))
        np.testing.assert_array_equal(k["st"][1][:S].view(np.uint32), w["st"])
        np.testing.assert_array_equal(k["voff"][1].view(np.uint64), w["voff"])
        np.testing.assert_array_equal(k["cs"][1].view(np.uint32), w["cs"])
        np.testing.assert_array_equal(k["se"][1][:s.n_entities_in_world].view(np.uint32), w["se"])

    s = chd.capi.TickSummary()
    prefetch(frames[0])
    enqueue(0)
    for i in range(1, len(frames)):
        enqueue(i)  # overwrites the engine's arrays while tick i-1's results are still travelling
        if i == 2:
            with pytest.raises(chd.capi.ChdError):  # two fetches outstanding: refused, nothing enqueued
                ck(e.L.chd_fetch_results_async(e.h, C.byref(sets[0][0]), chd.capi.ptr(sets[0][1]["hdr"][0])))
        ck(e.L.chd_fetch_wait(e.h, C.byref(s)))
        check(i - 1, s)
    ck(e.L.chd_fetch_wait(e.h, C.byref(s)))
    check(len(frames) - 1, s)
    assert sum(w["s"]["n_handover"] for w in want) > 100 and sum(w["s"]["n_due"] for w in want) > 1000
    with pytest.raises(chd.capi.ChdError):
        ck(e.L.chd_fetch_wait(e.h, C.byref(s)))  # nothing in flight
    e.close()


def test_zero_copy_device_inputs_match_host_inputs(chd):
    """Device-resident positions / queries / rings are consumed in place; results equal the host-input path."""
    import torch

    wc = chd.synth.scaled(chd.synth.CONFIGS["benchmark"], 40_000, 4_000)
    out = {}
    for mode in ("host", "device"):
        e = chd.engine.Engine(wc.cfg(), wc.n_entities, wc.n_subscribers, max_visible=1 << 23)
        ex, ez = chd.synth.entities(wc)
        conn, _, _, _ = chd.synth.subscribers(wc, ex, ez)
        e.set_subscribers(conn)
        ring_state, res = None, []
        keep = []
        for tick in range(5):
            t = (tick + 1) * 33_000_000
            ex, ez = chd.synth.move_entities(wc, ex, ez, tick, 300.0)
            _, cx, cz, r = chd.synth.subscribers(wc, ex, ez)
            ring_state, off, arr, snd, idx, cmi = chd.synth.update_rings(wc, tick, t, 33_000_000, 4, len(conn), ring_len=16, state=ring_state)
            if mode == "device":
                dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int64 if a.dtype.itemsize == 8 and a.dtype.kind != "f" else
                                                                               (np.int32 if a.dtype.kind != "f" else a.dtype))).cuda()
                tx, tz, tcx, tcz, tr = (torch.from_numpy(a).cuda() for a in (ex, ez, cx, cz, r))
                toff, tarr, tsnd, tidx, tcmi = dev(off), dev(arr), dev(snd), dev(idx), dev(cmi)
                keep.append((tx, tz, tcx, tcz, tr, toff, tarr, tsnd, tidx, tcmi))  # stay alive until consumed
                torch.cuda.synchronize()
                e._ck(e.L.chd_set_entities(e.h, tx.data_ptr(), tz.data_ptr(), len(ex)))
                e._ck(e.L.chd_set_rings(e.h, toff.data_ptr(), int(off[-1]), tarr.data_ptr(), tsnd.data_ptr(), tidx.data_ptr(), tcmi.data_ptr()))
                batch, k2 = chd.engine.make_batch(len(cx), sub=None, sphere=(tcx, tcz, tr))
            else:
                e.set_entities(ex, ez)
                e.set_rings(off, arr, snd, idx, cmi)
                batch, k2 = chd.engine.make_batch(len(cx), sub=None, sphere=(cx, cz, r))
            s = e.tick(batch, t, chd.capi.TICK_ALL)
            pairs = e.get_pairs(s.n_pairs)
            voff, vis = e.get_visible()
            due = e.get_due(s.n_due)
            due = due[np.lexsort((due["window_hi"], due["channel_id"], due["sub"]))]
            res.append((s.as_dict(), pairs, voff, vis, due))
        out[mode] = res
    for a, b in zip(out["host"], out["device"]):
        assert a[0] == b[0]
        for k in a[1]:
            np.testing.assert_array_equal(a[1][k], b[1][k])
        np.testing.assert_array_equal(a[2], b[2]); np.testing.assert_array_equal(a[3], b[3]); np.testing.assert_array_equal(a[4], b[4])
    assert sum(r[0]["n_due"] for r in out["host"]) > 1000


def test_prefetched_inputs_match_direct_upload(chd):
    """chd_prefetch_{entities,queries,rings} + chd_adopt_prefetched (double-buffered uploads that overlap the tick in
    flight) give the same pairs, visible lists, fan-out decisions and handover lists as chd_set_entities / chd_set_rings /
    an explicit query batch, tick after tick.  "mixed" switches between the two (a direct tick between prefetched ones) and
    prefetches one tick's inputs twice, the first time with other data: the second upload is the one adopted."""
    wc = chd.synth.scaled(chd.synth.CONFIGS["benchmark"], 60_000, 5_000)
    ex, ez = chd.synth.entities(wc)
    conn, _, _, _ = chd.synth.subscribers(wc, ex, ez)
    frames, ring_state = [], None
    for tick in range(7):
        t = (tick + 1) * 33_000_000
        ex, ez = chd.synth.move_entities(wc, ex, ez, tick, 400.0)
        _, cx, cz, r = chd.synth.subscribers(wc, ex, ez)
        ring_state, off, arr, snd, idx, cmi = chd.synth.update_rings(wc, tick, t, 33_000_000, 4, len(conn), ring_len=16, state=ring_state)
        frames.append(dict(t=t, x=ex.copy(), z=ez.copy(), q=(cx, cz, r), rings=(off, arr, snd, idx, cmi)))
    plans = {"direct": ["direct"] * 7, "prefetch": ["prefetch"] * 7,
             "mixed": ["prefetch", "prefetch", "direct", "prefetch", "prefetch", "twice", "prefetch"]}
    out = {}
    for mode, plan in plans.items():
        e = chd.engine.Engine(wc.cfg(), wc.n_entities, wc.n_subscribers, max_visible=1 << 24)
        e.set_subscribers(conn)
        res = []

        def prefetch(f, n=None):
            batch, keep = chd.engine.make_batch(len(f["q"][0]), sub=None, sphere=f["q"])
            e.prefetch_rings(*f["rings"])
            e.prefetch_queries(batch, keep)
            e.prefetch_entities(f["x"], f["z"], n)

        def stage(tick):  # uploads the inputs of a prefetched tick ahead of it
            if tick < len(frames) and plan[tick] != "direct":
                if plan[tick] == "twice":
                    prefetch(frames[0], len(frames[0]["x"]) - 1000)  # other positions (and fewer), queries and rings
                prefetch(frames[tick])

        stage(0)
        for tick, f in enumerate(frames):
            if plan[tick] == "direct":
                e.set_rings(*f["rings"])
                e.set_entities(f["x"], f["z"])
                batch, keep = chd.engine.make_batch(len(f["q"][0]), sub=None, sphere=f["q"])
                e.tick(batch, f["t"], chd.capi.TICK_ALL, want_summary=False)
            else:
                e.adopt_prefetched()
                e.begin_interest(None, f["t"])
                e.tick(None, f["t"], chd.capi.TICK_ALL | chd.capi.TICK_EARLY_RESULTS, want_summary=False)  # asynchronous
            stage(tick + 1)  # goes up while the tick runs
            s = e.summary()
            pairs = e.get_pairs(s.n_pairs)
            voff, vis = e.get_visible()
            due = e.get_due(s.n_due)
            due = due[np.lexsort((due["window_hi"], due["channel_id"], due["sub"]))]
            ho = np.stack(e.get_handover(s.n_handover), 1)
            ho = ho[np.lexsort((ho[:, 2], ho[:, 1], ho[:, 0]))]
            res.append((s.as_dict(), pairs, voff, vis, due, ho))
        with pytest.raises(Exception):
            e.adopt_prefetched()  # nothing staged any more
        with pytest.raises(Exception):
            e.begin_interest(None, 1)  # no adopted batch
        out[mode] = res
    for mode in ("prefetch", "mixed"):
        for a, b in zip(out["direct"], out[mode]):
            assert a[0] == b[0], mode
            for k in a[1]:
                np.testing.assert_array_equal(a[1][k], b[1][k])
            for i in (2, 3, 4, 5):
                np.testing.assert_array_equal(a[i], b[i])
    assert sum(r[0]["n_handover"] for r in out["direct"]) > 100 and sum(r[0]["n_due"] for r in out["direct"]) > 1000


def test_float_positions_match_widened_doubles(chd, oracle):
    """chd_set_entities_f32 / chd_prefetch_entities_f32 (positions that are FVector floats at the source, pkg/unrealpb/extension.go:10-24:
    info.X = float64(*vec.X)) give bit-identical results to chd_set_entities fed with the widened doubles, and to the oracle; odd
    entity counts exercise the kernel's scalar tail; device-resident float arrays are widened in place."""
    import torch

    wc = chd.synth.scaled(chd.synth.CONFIGS["benchmark"], 60_001, 5_000)
    og = _oracle_grid(wc)
    ex, ez = chd.synth.entities(wc)
    conn, _, _, _ = chd.synth.subscribers(wc, ex, ez)
    frames = []
    for tick in range(4):
        ex, ez = chd.synth.move_entities(wc, ex, ez, tick, 400.0)
        xf, zf = ex.astype(np.float32), ez.astype(np.float32)
        xd, zd = xf.astype(np.float64), zf.astype(np.float64)
        _, cx, cz, r = chd.synth.subscribers(wc, xd, zd)
        frames.append(dict(t=(tick + 1) * 33_000_000, xf=xf, zf=zf, xd=xd, zd=zd, q=(cx, cz, r)))
    out = {}
    for mode in ("f64", "f32", "f32_prefetch", "f32_device"):
        e = chd.engine.Engine(wc.cfg(), wc.n_entities, wc.n_subscribers, max_visible=1 << 24)
        e.set_subscribers(conn)
        res = []
        if mode == "f32_prefetch":
            e.prefetch_entities_f32(frames[0]["xf"], frames[0]["zf"])
        for tick, f in enumerate(frames):
            batch, keep = chd.engine.make_batch(len(f["q"][0]), sub=None, sphere=f["q"])
            if mode == "f64":
                e.set_entities(f["xd"], f["zd"])
            elif mode == "f32":
                e.set_entities_f32(f["xf"], f["zf"])
            elif mode == "f32_device":
                dx, dz = torch.from_numpy(f["xf"]).cuda(), torch.from_numpy(f["zf"]).cuda()
                torch.cuda.synchronize()
                e.set_entities_f32(dx, dz, len(f["xf"]))
            else:
                e.adopt_prefetched()
                if tick + 1 < len(frames):
                    e.prefetch_entities_f32(frames[tick + 1]["xf"], frames[tick + 1]["zf"])
            s = e.tick(batch, f["t"], chd.capi.TICK_ALL)
            pairs = e.get_pairs(s.n_pairs)
            voff, vis = e.get_visible()
            ho = np.stack(e.get_handover(s.n_handover), 1)
            ho = ho[np.lexsort((ho[:, 2], ho[:, 1], ho[:, 0]))]
            res.append((s.as_dict(), pairs, voff, vis, ho))
        out[mode] = res
        e.close()
    for mode in ("f32", "f32_prefetch", "f32_device"):
        for a, b in zip(out["f64"], out[mode]):
            assert a[0] == b[0], mode
            for k in a[1]:
                np.testing.assert_array_equal(a[1][k], b[1][k])
            for i in (2, 3, 4):
                np.testing.assert_array_equal(a[i], b[i])
    f = frames[-1]
    want = oracle.sphere_tick(og, f["xd"], f["zd"], *f["q"])
    np.testing.assert_array_equal(out["f32"][-1][1]["channel"], want["pair_cell"])
    np.testing.assert_array_equal(out["f32"][-1][3], want["vis_entity"])
    assert sum(r[0]["n_handover"] for r in out["f64"]) > 100


def test_adjacent_broadcast_sets_parity(chd, oracle):
    """BroadcastType_ADJACENT_CHANNELS recipient sets (message.go:188-239) for a batch of messages against the oracle
    restatement: every cell x every filter combination + random senders / forwarded clients, on subscriptions built
    by chd_update_interest from random sphere queries (many subscribers span several cells, so the de-duplication is
    exercised); also the empty / invalid-channel / capacity edges."""
    from tests._oracle import make_grid

    g = GRIDS[5]  # 9 x 8 grid, 100 x 50 cells
    og = make_grid(*g)
    cells = 72
    rng = np.random.default_rng(99)
    S = 3000
    e = chd.engine.Engine(chd.engine.grid_cfg(*g), 16, S, max_visible=1 << 16)
    e.set_entities(np.array([0.0]), np.array([0.0]))
    e.build()
    conn = (rng.permutation(S) + 1).astype(np.uint32)
    types = rng.integers(1, 3, S).astype(np.uint8)
    e.set_subscribers(conn)
    # nothing subscribed yet: every list is empty
    st, off, slot = e.adjacent_broadcast([S0 + 3, S0 + 40], [64, 64])
    assert st.tolist() == [0, 0] and off.tolist() == [0, 0, 0] and len(slot) == 0
    e.set_subscriber_types(types)
    cx, cz = rng.uniform(-450, 450, S), rng.uniform(-200, 200, S)
    r = rng.choice([10.0, 40.0, 90.0, 160.0], S)
    batch, keep = chd.engine.make_batch(S, sub=None, sphere=(cx, cz, r))
    for tick in range(2):  # second update: pairs live in the other buffer, by-cell order rebuilt
        if tick == 1:
            cx = cx + rng.uniform(-30, 30, S)
            batch, keep = chd.engine.make_batch(S, sub=None, sphere=(cx, cz, r))
        e.update_interest(batch, (tick + 1) * 1000 * MS)
        s = e.summary()
        pairs = e.get_pairs(s.n_pairs)
        # every channel's subscriber list from the engine's (already parity-checked) pairs
        sub_of_pair = np.repeat(np.arange(S), np.diff(pairs["off"].astype(np.int64)))
        cell_of_pair = pairs["channel"].astype(np.int64) - S0
        order = np.lexsort((sub_of_pair, cell_of_pair))
        cell_off = np.searchsorted(cell_of_pair[order], np.arange(cells + 1)).astype(np.uint32)
        list_conn, list_type = conn[sub_of_pair[order]], types[sub_of_pair[order]]
        assert (np.diff(pairs["off"].astype(np.int64)) > 1).sum() > S // 10  # plenty of multi-cell subscribers
        combos = [0, 4, 8, 16, 32, 4 | 8, 8 | 16, 8 | 32, 4 | 16 | 32, 2]
        ch, fl, snd, cli = [], [], [], []
        for c in range(cells):
            for f in combos:
                ch.append(S0 + c); fl.append(64 | f)
                snd.append(int(conn[rng.integers(0, S)]) if rng.random() < 0.8 else 0)
                cli.append(int(conn[rng.integers(0, S)]) if rng.random() < 0.5 else 0)
        ch += [S0 + cells, S0 - 1, 5]  # not cells of this grid
        fl += [64, 64, 64]; snd += [0, 0, 0]; cli += [0, 0, 0]
        st, off, slot = e.adjacent_broadcast(ch, fl, snd, cli)
        assert st[-3:].tolist() == [1, 1, 1] and (st[:-3] == 0).all()
        assert off[-4] == off[-1]  # invalid channels get no recipients
        n_multi = 0
        for m in range(len(ch) - 3):
            got = conn[slot[off[m]:off[m + 1]]]
            assert len(np.unique(got)) == len(got), "a connection was reported twice"
            want = oracle.adjacent_broadcast(og, ch[m], fl[m], snd[m], cli[m], cell_off, list_conn, list_type)
            np.testing.assert_array_equal(np.sort(got), want)
            n_multi += len(got)
        assert n_multi > 50_000
        # without types the client / server filters remove nobody
        e.set_subscriber_types(None)
        st2, off2, slot2 = e.adjacent_broadcast([S0 + 40, S0 + 40], [64 | 16, 64])
        np.testing.assert_array_equal(np.sort(slot2[off2[0]:off2[1]]), np.sort(slot2[off2[1]:off2[2]]))
        e.set_subscriber_types(types)
        # capacity is an error, never a truncation
        with pytest.raises(Exception):
            e.adjacent_broadcast(ch[:50], fl[:50], cap=3)


def test_update_interest_all_aoi_kinds(chd, oracle):
    """The stateful path (chd_update_interest) with spots / box / sphere / cone queries and their combinations:
    every subscriber's subscription set (channel, dist, damping interval) equals the oracle's QueryChannelIds; failed
    queries leave the previous subscriptions untouched (message_spatial.go:60-63)."""
    from tests._oracle import make_grid

    g = GRIDS[5]  # 9 x 8 grid, 100 x 50 cells
    og = make_grid(*g)
    rng = np.random.default_rng(4242)
    S = 600
    e = chd.engine.Engine(chd.engine.grid_cfg(*g), 16, S, max_spots=1 << 14, max_window_cells=1 << 20, max_visible=1 << 16)
    e.set_entities(np.array([0.0]), np.array([0.0]))
    e.build()
    e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
    state = [dict() for _ in range(S)]
    for tick in range(3):
        qs = _random_queries(rng, g, S)
        order = rng.permutation(S)  # query i belongs to subscriber order[i]
        batch, keep = chd.controller.pack_queries(qs, subs=order.astype(np.uint32))
        e.update_interest(batch, (tick + 1) * 33_000_000)
        s = e.summary()
        status = e.get_query_status(S)
        n_err = 0
        for i, q in enumerate(qs):
            want, st = _oracle_query(oracle, og, q)
            if st != 0:
                n_err += 1
                assert status[i] != 0
            else:
                assert status[i] == 0
                state[order[i]] = want
        assert s.n_query_errors == n_err and 0 < n_err < S
        pairs = e.get_pairs(s.n_pairs)
        for j in range(S):
            sl = slice(pairs["off"][j], pairs["off"][j + 1])
            got = dict(zip(pairs["channel"][sl].tolist(), pairs["dist"][sl].tolist()))
            assert got == state[j], (tick, j)
            assert pairs["interval"][sl].tolist() == [oracle.damping(d, 20) for d in pairs["dist"][sl].tolist()]


def test_concurrent_stateless_queries_during_ticks(chd, oracle):
    """GetChannelId / QueryChannelIds are called from arbitrary channel goroutines while the tick driver runs
    (spatial.go:20-29): a second thread hammers the stateless entry points during batched ticks; both stay exact."""
    import threading

    wc = chd.synth.scaled(chd.synth.CONFIGS["benchmark"], 50_000, 5_000)
    og = _oracle_grid(wc)
    e = chd.engine.Engine(wc.cfg(), wc.n_entities, wc.n_subscribers, max_visible=1 << 23)
    ex, ez = chd.synth.entities(wc)
    conn, cx, cz, r = chd.synth.subscribers(wc, ex, ez)
    e.set_subscribers(conn)
    stop, errors = threading.Event(), []

    def worker():
        rng = np.random.default_rng(7)
        while not stop.is_set():
            try:
                x, z = rng.uniform(-16000, 16000, 257), rng.uniform(-16000, 16000, 257)
                if not np.array_equal(e.cell_of(x, z), oracle.cell_of(og, x, z)):
                    errors.append("cell_of mismatch")
                n = 64
                qx, qz, qr = rng.uniform(-15000, 15000, n), rng.uniform(-15000, 15000, n), rng.choice([50.0, 900.0, 2500.0], n)
                b, keep = chd.engine.make_batch(n, sphere=(qx, qz, qr))
                st, off, ids, dist = e.query_channel_ids(b)
                for i in range(n):
                    want, wst = oracle.query(og, sphere=(qx[i], qz[i], qr[i]))
                    got = dict(zip(ids[off[i]:off[i + 1]].tolist(), dist[off[i]:off[i + 1]].tolist()))
                    if (wst != 0) != (st[i] != 0) or (wst == 0 and got != want):
                        errors.append("query mismatch")
            except Exception as ex_:  # noqa: BLE001
                errors.append(repr(ex_))
                return

    th = threading.Thread(target=worker)
    th.start()
    try:
        for tick in range(30):
            ex, ez = chd.synth.move_entities(wc, ex, ez, tick, 200.0)
            _, cx, cz, r = chd.synth.subscribers(wc, ex, ez)
            e.set_entities(ex, ez)
            batch, keep = chd.engine.make_batch(len(cx), sub=None, sphere=(cx, cz, r))
            s = e.tick(batch, (tick + 1) * 33_000_000, chd.capi.TICK_BUILD | chd.capi.TICK_EMIT)
            if tick % 10 == 9:
                want = oracle.sphere_tick(og, ex, ez, cx, cz, r)
                pairs = e.get_pairs(s.n_pairs)
                voff, vis = e.get_visible()
                np.testing.assert_array_equal(pairs["channel"], want["pair_cell"])
                np.testing.assert_array_equal(voff, want["vis_off"])
                np.testing.assert_array_equal(vis, want["vis_entity"])
    finally:
        stop.set()
        th.join(60)
    assert not errors, errors[:3]


def test_emit_descriptor_base_wraps_below_zero(chd, oracle):
    """A tile whose second segment is a cell that starts EARLIER in the CSR than the first segment ends in the tile: the descriptor's
    second base is stored minus that end and wraps below zero (32-bit arithmetic on purpose).  With the two ends congruent mod 4 the
    second segment's chunks are aligned 16-byte loads of the sorted array and the 16-byte chunk across the boundary goes entry
    by entry — the combination that used to be added in 64 bits (out-of-bounds read)."""
    wc = chd.synth.CONFIGS["2x2"]
    og = _oracle_grid(wc)
    centres = [(wc.offx + (c + 0.5) * wc.w, wc.offz + (r + 0.5) * wc.h) for r in range(wc.rows) for c in range(wc.cols)]
    ids = oracle.cell_of(og, np.array([c[0] for c in centres]), np.array([c[1] for c in centres]))
    centres = [centres[k] for k in np.argsort(ids)]  # ascending cell index = CSR order
    counts = [1001, 5000, 8192 + 2005, 0]  # cell 1 starts at 1001; the big cell ends 2005 entries into the tile that starts at 8192: 2005 % 4 == 1001 % 4
    rng = np.random.default_rng(5)
    xs, zs = [], []
    for (cx_, cz_), n in zip(centres, counts):
        xs.append(cx_ + rng.uniform(-0.4, 0.4, n) * wc.w)
        zs.append(cz_ + rng.uniform(-0.4, 0.4, n) * wc.h)
    ex, ez = np.concatenate(xs), np.concatenate(zs)
    perm = rng.permutation(len(ex))
    ex, ez = ex[perm], ez[perm]
    # subscriber 0 sees the big cell only, subscriber 1 the 5000-entity cell only
    cx = np.array([centres[2][0], centres[1][0]])
    cz = np.array([centres[2][1], centres[1][1]])
    r = np.array([50.0, 50.0])
    e = chd.engine.Engine(wc.cfg(), len(ex), 2, max_visible=1 << 20)
    e.set_entities(ex, ez)
    e.set_subscribers(np.array([11, 12], np.uint32))
    batch, keep = chd.engine.make_batch(2, sub=None, sphere=(cx, cz, r))
    for tick in range(3):  # direct launches, then the replayed graphs
        s = e.tick(batch, (tick + 1) * 33_000_000, chd.capi.TICK_BUILD | chd.capi.TICK_EMIT)
        want = oracle.sphere_tick(og, ex, ez, cx, cz, r)
        voff, vis = e.get_visible()
        np.testing.assert_array_equal(voff, want["vis_off"])
        np.testing.assert_array_equal(vis, want["vis_entity"])
        assert s.n_visible == counts[2] + counts[1]
    e.close()


def test_full_size_config2_properties(chd, oracle):
    """BASELINE config #2 at FULL size (1 M entities / 100 K subscribers, r = 50): size-independent properties of the
    whole result + bit-exact oracle comparison on a 2 % subscriber sample."""
    wc = chd.synth.CONFIGS["benchmark"]
    ex, ez = chd.synth.entities(wc)
    conn, cx, cz, r = chd.synth.subscribers(wc, ex, ez)
    S, N = wc.n_subscribers, wc.n_entities
    e = chd.engine.Engine(wc.cfg(), N, S, max_visible=int(6.0e8))
    e.set_entities(ex, ez)
    e.set_subscribers(conn)
    batch, keep = chd.engine.make_batch(S, sub=None, sphere=(cx, cz, r))
    s = e.tick(batch, 33_000_000, chd.capi.TICK_BUILD | chd.capi.TICK_EMIT)
    # cell CSR: a permutation of the in-world entities, sorted by (cell, entity id)
    cs, se = e.get_cells()
    ids = oracle.cell_of(_oracle_grid(wc), ex, ez)
    in_world = ids != 0
    assert s.n_entities_in_world == int(in_world.sum()) == len(se) == int(cs[-1])
    assert int(se.astype(np.uint64).sum()) == int(np.nonzero(in_world)[0].astype(np.uint64).sum())  # checksum: every id once
    cell_of_sorted = ids[se] - S0
    assert (np.diff(cell_of_sorted.astype(np.int64)) >= 0).all()  # sorted by cell
    same = np.diff(cell_of_sorted.astype(np.int64)) == 0
    assert (np.diff(se.astype(np.int64))[same] > 0).all()  # entity ids ascending inside a cell
    np.testing.assert_array_equal(cs, np.concatenate([[0], np.cumsum(np.bincount(cell_of_sorted, minlength=wc.cells))]))
    # pairs / visible lists: totals are consistent with the CSR
    pairs = e.get_pairs(s.n_pairs)
    voff = np.zeros(S + 1, np.uint64)
    e._ck(e.L.chd_get_visible(e.h, chd.capi.ptr(voff), None))
    counts = np.diff(cs.astype(np.int64))
    per_pair = counts[pairs["channel"] - S0]
    per_sub = np.add.reduceat(per_pair, pairs["off"][:-1].astype(np.int64)) if s.n_pairs else np.zeros(S)
    per_sub[np.diff(pairs["off"].astype(np.int64)) == 0] = 0
    np.testing.assert_array_equal(np.diff(voff.astype(np.int64)), per_sub)
    assert s.n_visible == int(voff[-1]) == int(per_pair.sum()) > 4.0e8
    assert (pairs["dist"] <= 1).all() and s.n_query_errors == int((e.get_query_status(S) != 0).sum())
    # 2 % sample against the oracle, bit-exact (pairs, dists, visible lists)
    sel = np.linspace(0, S - 1, S // 50).astype(np.int64)
    want = oracle.sphere_tick(_oracle_grid(wc), ex, ez, cx[sel], cz[sel], r[sel])
    for k, j in enumerate(sel):
        a = slice(pairs["off"][j], pairs["off"][j + 1])
        b = slice(int(want["pair_off"][k]), int(want["pair_off"][k + 1]))
        np.testing.assert_array_equal(pairs["channel"][a], want["pair_cell"][b])
        np.testing.assert_array_equal(pairs["dist"][a], want["pair_dist"][b])
        np.testing.assert_array_equal(e.get_visible_slot(int(j)), want["vis_entity"][int(want["vis_off"][k]):int(want["vis_off"][k + 1])])


@pytest.mark.parametrize("name", ["10m", "handover"])
def test_full_size_configs_3_and_5(chd, oracle, name):
    """BASELINE configs #3 (64x64 grid) and #5 (256x256 grid of 100x100 cells, hash rebuilt every tick, half of the entities
    changing cell) at FULL size — 10 M entities / 1 M subscribers, the 2-pass radix build — over two ticks: size-independent
    properties of the whole result (CSR is a sorted permutation, offsets consistent, handover list = entities whose cell changed)
    and a bit-exact oracle comparison of a 0.1 % subscriber sample on both ticks."""
    wc = chd.synth.CONFIGS[name]
    S, N = wc.n_subscribers, wc.n_entities
    ex, ez = chd.synth.entities(wc)
    og = _oracle_grid(wc)
    per_cell = N / wc.cells
    e = chd.engine.Engine(wc.cfg(), N, S, max_visible=int(S * 1.15 * per_cell * (1.0 + 4.0 * wc.radius / wc.w) + (1 << 22)))
    conn = np.arange(1, S + 1, dtype=np.uint32)
    e.set_subscribers(conn)
    prev_ids = None
    for tick in range(2):
        if tick == 1:
            if name == "handover":  # SURVEY §8d #5: a seeded half of the entities jumps one cell in a random axis direction
                i = np.arange(N, dtype=np.uint64)
                jump = chd.synth.uniform(wc.seed + 50, i, 0) < 0.5
                axis = chd.synth.uniform(wc.seed + 51, i, 0) < 0.5
                sign = np.where(chd.synth.uniform(wc.seed + 52, i, 0) < 0.5, -1.0, 1.0)
                ex = np.where(jump & axis, ex + sign * wc.w, ex)
                ez = np.where(jump & ~axis, ez + sign * wc.h, ez)
            else:
                ex, ez = chd.synth.move_entities(wc, ex, ez, 1, 60.0)
        _, cx, cz, r = chd.synth.subscribers(wc, ex, ez)
        e.set_entities(ex, ez)
        batch, keep = chd.engine.make_batch(S, sub=None, sphere=(cx, cz, r))
        s = e.tick(batch, (tick + 1) * 33_000_000, chd.capi.TICK_BUILD | chd.capi.TICK_EMIT)
        assert s.overflow == 0
        cs, se = e.get_cells()
        ids = oracle.cell_of(og, ex, ez)
        in_world = ids != 0
        assert s.n_entities_in_world == int(in_world.sum()) == len(se) == int(cs[-1])
        assert int(se.astype(np.uint64).sum()) == int(np.nonzero(in_world)[0].astype(np.uint64).sum())
        cell_of_sorted = (ids[se] - S0).astype(np.int64)
        d = np.diff(cell_of_sorted)
        assert (d >= 0).all() and (np.diff(se.astype(np.int64))[d == 0] > 0).all()
        np.testing.assert_array_equal(cs, np.concatenate([[0], np.cumsum(np.bincount(cell_of_sorted, minlength=wc.cells))]))
        if prev_ids is not None:  # handover candidates = entities whose GetChannelId changed (spatial.go:612-626)
            moved = np.nonzero(prev_ids != ids)[0]
            assert s.n_handover == len(moved)
            he, hs, hd = e.get_handover(s.n_handover)
            order = np.argsort(he)
            np.testing.assert_array_equal(he[order], moved)
            np.testing.assert_array_equal(hs[order], prev_ids[moved])
            np.testing.assert_array_equal(hd[order], ids[moved])
            if name == "handover":
                assert len(moved) > 0.45 * N
        prev_ids = ids
        pairs = e.get_pairs(s.n_pairs)
        voff = np.zeros(S + 1, np.uint64)
        e._ck(e.L.chd_get_visible(e.h, chd.capi.ptr(voff), None))
        counts = np.diff(cs.astype(np.int64))
        per_pair = counts[pairs["channel"] - S0]
        assert s.n_visible == int(voff[-1]) == int(per_pair.sum())
        sel = np.linspace(0, S - 1, S // 1000).astype(np.int64)
        want = oracle.sphere_tick(og, ex, ez, cx[sel], cz[sel], r[sel])
        for k, j in enumerate(sel):
            a = slice(pairs["off"][j], pairs["off"][j + 1])
            b = slice(int(want["pair_off"][k]), int(want["pair_off"][k + 1]))
            np.testing.assert_array_equal(pairs["channel"][a], want["pair_cell"][b])
            np.testing.assert_array_equal(pairs["dist"][a], want["pair_dist"][b])
            np.testing.assert_array_equal(e.get_visible_slot(int(j)), want["vis_entity"][int(want["vis_off"][k]):int(want["vis_off"][k + 1])])
    e.close()
