"""Followers and explicit queries in one interest update (chd_follow_queries_with): the host's batch merged in front of the generated
follower batch on the device.  The reference for every check is a second engine fed the host-packed equivalent through the ordinary
query path: the host part, skip entries up to its size class H, the followers' queries (overridden slots left out), skip entries up
to H + B.
Run on an H100:  python -m pytest tests -m gpu"""
import ctypes as C

import numpy as np
import pytest

from tests.test_gpu_follow import TICK, World, assert_same, refused, rings, snapshot

gpu = pytest.mark.gpu
SPOTS, BOX, SPHERE, CONE = 1, 2, 4, 8
SKIP = 0xFFFFFFFF


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
    ns.capi, ns.engine, ns.synth, ns.torch = capi, engine, synth, torch
    return ns


FIELDS = ("sph_cx", "sph_cz", "sph_r", "box_cx", "box_cz", "box_ex", "box_ez", "cone_cx", "cone_cz", "cone_dx", "cone_dz", "cone_angle", "cone_r")
GROUPS = {SPHERE: FIELDS[0:3], BOX: FIELDS[3:7], CONE: FIELDS[7:13]}


class Part:
    """A query batch as numpy arrays: sub, kind (None: all sphere), the 13 f64 arrays (absent ones None) and the spots (or None)."""

    def __init__(self, sub, kind, f, spots=None):
        self.sub, self.kind, self.f, self.spots = np.asarray(sub, np.uint32), kind, f, spots

    @property
    def n(self):
        return len(self.sub)

    def batch(self, engine):
        g = lambda *ks: None if self.f[ks[0]] is None else tuple(self.f[k] for k in ks)
        return engine.make_batch(self.n, sub=self.sub, kind=self.kind, sphere=g(*GROUPS[SPHERE]), box=g(*GROUPS[BOX]), cone=g(*GROUPS[CONE]),
                                 spots=self.spots)


def host_part(W, n, slots, spots=True, omit=(), bad_kind_rows=(), spots_per=(1, 5)):
    """n explicit queries for the given slots: every kind (spots too), centres anywhere in the world, not on a pawn.  omit: kinds whose
    arrays the part does not supply (no entry uses them unless listed in bad_kind_rows, whose kind gets them added).  An entry with
    CHD_AOI_SPOTS has spots_per[0] to spots_per[1] - 1 spots."""
    rng = W.rng
    kinds = [SPHERE, BOX, CONE, SPOTS, SPHERE | SPOTS, BOX | CONE, SPHERE | BOX | CONE | SPOTS, SPHERE | 0x40]  # (a stray high bit)
    if not spots:
        kinds = [k & ~SPOTS or SPHERE for k in kinds]
    usable = [k for k in kinds if not any(k & o for o in omit)]
    kind = np.array([usable[i % len(usable)] for i in range(n)], np.uint8)
    for r in bad_kind_rows:
        kind[r] |= omit[0]
    wx, wz = W.cols * W.w, W.rows * W.w
    cx, cz = rng.uniform(0, wx, n), rng.uniform(0, wz, n)
    ang = rng.uniform(0, 2 * np.pi, n)
    f = dict(sph_cx=cx, sph_cz=cz, sph_r=rng.uniform(5, 120, n), box_cx=cx + 1, box_cz=cz - 1, box_ex=rng.uniform(5, 90, n),
             box_ez=rng.uniform(5, 90, n), cone_cx=cx, cone_cz=cz, cone_dx=np.cos(ang), cone_dz=np.sin(ang), cone_angle=rng.uniform(0.2, 1.2, n),
             cone_r=rng.uniform(20, 150, n))
    for o in omit:
        for k in GROUPS[o]:
            f[k] = None
    sp = None
    if spots:
        cnt = np.where(kind & SPOTS, rng.integers(spots_per[0], spots_per[1], n), 0)
        off = np.zeros(n + 1, np.uint32)
        off[1:] = np.cumsum(cnt)
        t = int(off[-1])
        sp = (off, rng.integers(0, 5, n).astype(np.uint32), rng.uniform(0, wx, t), rng.uniform(0, wz, t), rng.integers(0, 4, t).astype(np.uint32))
    return Part(np.asarray(slots, np.uint32)[:n], kind, f, sp)


def pick_slots(rng, n, S, followers, frac_override=0.3, unknown=True):
    """n distinct slots: about frac_override of them following slots (overrides), one unknown slot (>= S) when n > 2"""
    fol = rng.permutation(np.asarray(sorted(followers), np.int64))
    free = rng.permutation(np.setdiff1d(np.arange(S), fol))
    k = min(int(n * frac_override), len(fol))
    out = np.concatenate([fol[:k], free[:n - k]])
    if unknown and n > 2:
        out[-1] = S + 3
    return rng.permutation(out).astype(np.uint32)[:n]


class Follow:
    """The followers' side of the mirror: CHD_FOLLOW_ALL / MOVED selection with overrides, and what chd_get_follow reports."""

    def __init__(self, W):
        self.W = W
        self.last = {}
        self.dirty = set()

    def bound(self, slots):
        for s in slots:
            self.last[int(s)] = (0.0, 0.0)
            self.dirty.add(int(s))

    def generate(self, mode, overridden):
        W, sel, status = self.W, [], {}
        for s in sorted(W.bind):
            p = W.bind[s][0]
            if s in overridden:
                self.dirty.add(s)
                status[s] = 18
                continue
            if not W.live[p]:
                self.dirty.add(s)
                status[s] = 17
                continue
            x, z = float(W.x[p]), float(W.z[p])
            if mode == 1 and s not in self.dirty and (x, z) == self.last[s]:
                status[s] = 16
                continue
            self.last[s] = (x, z)
            self.dirty.discard(s)
            status[s] = None  # the query's status
            sel.append(s)
        return sel, status

    def part(self, sel, B):
        """the selected followers' queries (ascending slot order) and skip entries up to B"""
        W = self.W
        m = len(sel)
        sub = np.full(B, SKIP, np.uint32)
        sub[:m] = sel
        kind = np.zeros(B, np.uint8)
        f = {k: np.zeros(B) for k in FIELDS}
        for j, s in enumerate(sel):
            p, k, sh = W.bind[s]
            kind[j] = k
            x, z = self.last[s]
            f["sph_cx"][j] = f["box_cx"][j] = f["cone_cx"][j] = x
            f["sph_cz"][j] = f["box_cz"][j] = f["cone_cz"][j] = z
            f["sph_r"][j], f["box_ex"][j], f["box_ez"][j], f["cone_dx"][j], f["cone_dz"][j], f["cone_angle"][j], f["cone_r"][j] = sh
        return Part(sub, kind, f)


def packed(chd, host, H, fol):
    """The host-packed equivalent of a merged batch: host part, skip entries to H, the follower part."""
    n = host.n
    sub = np.concatenate([host.sub, np.full(H - n, SKIP, np.uint32), fol.sub])
    hk = host.kind if host.kind is not None else np.full(n, SPHERE, np.uint8)
    kind = np.concatenate([hk, np.zeros(H - n, np.uint8), fol.kind])
    f = {k: np.concatenate([host.f[k] if host.f[k] is not None else np.zeros(n), np.zeros(H - n), fol.f[k]]) for k in FIELDS}
    sp = None
    if host.spots is not None:
        off, nd, x, z, d = host.spots
        tail = len(sub) - n
        sp = (np.concatenate([off, np.full(tail, off[-1], np.uint32)]), np.concatenate([nd, np.zeros(tail, np.uint32)]), x, z, d)
    return Part(sub, kind, f, sp).batch(chd.engine)


def check_follow(fe, F, status, ref_status, H, sel):
    f = fe.get_follow()
    W = F.W
    sl = sorted(W.bind)
    np.testing.assert_array_equal(f["slot"], np.array(sl, np.uint32))
    rank = {s: j for j, s in enumerate(sel)}
    want = [status[s] if status[s] is not None else int(ref_status[H + rank[s]]) for s in sl]
    np.testing.assert_array_equal(f["status"], np.array(want, np.uint32))
    np.testing.assert_array_equal(f["cx"], np.array([F.last[s][0] for s in sl]))
    np.testing.assert_array_equal(f["cz"], np.array([F.last[s][1] for s in sl]))
    assert f["n_selected"] == len(sel)
    return f


@gpu
@pytest.mark.parametrize("table", [False, True], ids=["index", "table"])
@pytest.mark.parametrize("mix", [False, True], ids=["sphere", "mixed"])
@pytest.mark.parametrize("graphs", [True, False], ids=["graphs", "direct"])
@pytest.mark.parametrize("mode", [0, 1], ids=["all", "moved"])
def test_merged_equals_host_packed_batch(chd, table, mix, graphs, mode):
    """12 ticks of moving entities with rings and fan-out, host parts of every kind (spots too) whose size varies within and across
    size classes (0 included) and that override some followers: every result and status equals the host-packed engine's."""
    capi, engine = chd.capi, chd.engine
    W = World(chd, 4000, table=table)
    S = 900
    lim = dict(max_pairs=1 << 17, max_queries=S + 1024, max_spots=1 << 14)
    fe, he = W.engine(S, **lim), W.engine(S, **lim)
    for e in (fe, he):
        e.enable_graphs(graphs)
    slots = np.arange(0, S, 3, dtype=np.uint32)
    ent = W.rng.permutation(W.n)[:len(slots)]
    kind, shape = W.shapes(slots, mix)
    W.follow(fe, slots, ent, kind, shape)
    F = Follow(W)
    F.bound(slots)
    B = len(slots)
    sizes = [40, 100, 200, 250, 0, 300, 400, 500, 30, 60, 70, 90]
    state = None
    for t, n_h in enumerate(sizes, 1):
        if t > 1:
            W.step((fe, he), frac=0.3)
        state, off, arr, snd, idx, cmi = rings(chd, W, t, S, state)
        for e in (fe, he):
            e.set_rings(off, arr, snd, idx, cmi)
        host = host_part(W, n_h, pick_slots(W.rng, n_h, S, W.bind), spots=True)
        H = engine.host_part_size(n_h)
        hb, hkeep = host.batch(engine)
        g0 = fe.graph_launch_count()
        fe.follow_queries_with(mode, hb)
        g_follow = fe.graph_launch_count() - g0
        overridden = {int(s) for s in host.sub if int(s) in W.bind}
        sel, status = F.generate(mode, overridden)
        g0 = fe.graph_launch_count()
        fe.begin_interest(None, t * TICK, False)
        g_interest = fe.graph_launch_count() - g0
        sf = fe.tick(None, t * TICK, capi.TICK_ALL)
        rb, rkeep = packed(chd, host, H, F.part(sel, B))
        sh = he.tick(rb, t * TICK, capi.TICK_ALL)
        assert_same(snapshot(fe, sf), snapshot(he, sh), "tick %d" % t)
        rs = he.get_query_status(H + B)
        np.testing.assert_array_equal(fe.get_query_status(H + B), rs)
        check_follow(fe, F, status, rs, H, sel)
        assert sum(v == 18 for v in status.values()) == len(overridden) and (n_h == 0 or overridden)
        if graphs:
            # the follow stage replays once its key (H among them) was seen a tick before; the interest stage's key also holds the
            # pair-buffer parity, so it replays when H equals that of two ticks before
            if t > 1 and H == engine.host_part_size(sizes[t - 2]):
                assert g_follow == 1, (t, g_follow)
            if t > 2 and H == engine.host_part_size(sizes[t - 3]) and H == engine.host_part_size(sizes[t - 2]):
                assert g_interest == 2, (t, g_interest)
        else:
            assert g_follow == 0 and g_interest == 0
    assert sf.n_due > 0 and sf.n_kept > 0
    fe.close(), he.close()


@gpu
def test_override_is_undone_by_the_next_moved_generation(chd):
    """An overridden follower whose entity stands still is selected by the next MOVED generation, and its pairs return to exactly the
    follow shape's."""
    capi, engine = chd.capi, chd.engine
    W = World(chd, 2000)
    S = 64
    fe = W.engine(S, max_queries=S + 512)
    slots = np.arange(S, dtype=np.uint32)
    ent = np.arange(S) * 7
    kind, shape = W.shapes(slots, True)
    W.follow(fe, slots, ent, kind, shape)
    fe.follow_queries(capi.FOLLOW_ALL)
    fe.tick(None, TICK, capi.TICK_BUILD | capi.TICK_FOLLOW)
    p0 = fe.get_pairs()
    # slot 9 sends a far-away box this tick
    hb, keep = engine.make_batch(1, sub=np.array([9], np.uint32), kind=np.array([BOX], np.uint8),
                                 box=(np.array([750.0]), np.array([40.0]), np.array([30.0]), np.array([30.0])))
    fe.follow_queries_with(capi.FOLLOW_MOVED, hb)
    s = fe.tick(None, 2 * TICK, capi.TICK_BUILD | capi.TICK_FOLLOW)
    f = fe.get_follow()
    assert f["status"][9] == capi.FOLLOW_OVERRIDDEN and f["n_selected"] == 0 and s.n_unsub > 0
    assert f["cx"][9] == W.x[ent[9]] and f["cz"][9] == W.z[ent[9]]  # the stored centre stays
    p1 = fe.get_pairs()
    assert not np.array_equal(p1["channel"][p1["off"][9]:p1["off"][10]], p0["channel"][p0["off"][9]:p0["off"][10]])
    # nobody moved: MOVED selects exactly the overridden follower, and slot 9's pairs are the follow shape's again
    fe.follow_queries(capi.FOLLOW_MOVED)
    fe.tick(None, 3 * TICK, capi.TICK_BUILD | capi.TICK_FOLLOW)
    f = fe.get_follow()
    assert f["n_selected"] == 1 and f["status"][9] == 0
    assert (f["status"][np.arange(S) != 9] == capi.FOLLOW_NOT_SELECTED).all()
    p2 = fe.get_pairs()
    for k in ("off", "channel", "dist"):
        np.testing.assert_array_equal(p2[k], p0[k])
    fe.close()


@gpu
@pytest.mark.parametrize("omit", [CONE, BOX, SPHERE], ids=["cone", "box", "sphere"])
def test_host_entries_without_their_arrays(chd, omit):
    """Host entries whose kind names arrays the host part omitted get CHD_Q_ERR_MISSING_ARRAY although the followers supply that
    kind, and keep their subscriptions; the rest equals a reference batch in which those entries fail (an invalid radius)."""
    capi, engine = chd.capi, chd.engine
    W = World(chd, 3000)
    S = 400
    lim = dict(max_queries=S + 512, max_spots=1 << 12)
    fe, he = W.engine(S, **lim), W.engine(S, **lim)
    slots = np.arange(0, S, 2, dtype=np.uint32)
    ent = W.rng.permutation(W.n)[:len(slots)]
    kind, shape = W.shapes(slots, True)  # every shape kind among the followers
    W.follow(fe, slots, ent, kind, shape)
    F = Follow(W)
    F.bound(slots)
    B = len(slots)
    host_slots = pick_slots(W.rng, 60, S, W.bind, unknown=False)
    for t in (1, 2, 3):
        host = host_part(W, 60, host_slots, omit=(omit,), bad_kind_rows=(3, 17, 40) if t > 1 else ())
        hb, keep = host.batch(engine)
        fe.follow_queries_with(capi.FOLLOW_ALL, hb)
        sel, status = F.generate(capi.FOLLOW_ALL, {int(s) for s in host.sub if int(s) in W.bind})
        sf = fe.tick(None, t * TICK, capi.TICK_ALL | capi.TICK_FOLLOW)
        ref = Part(host.sub, host.kind.copy(), {k: (v.copy() if v is not None else np.zeros(host.n)) for k, v in host.f.items()}, host.spots)
        bad = [3, 17, 40] if t > 1 else []
        for r in bad:  # fails in the reference too, and keeps the subscriptions: a zero radius outside the world (no cell window)
            ref.kind[r] = SPHERE
            ref.f["sph_cx"][r], ref.f["sph_cz"][r], ref.f["sph_r"][r] = -1e6, -1e6, 0.0
        H = engine.host_part_size(host.n)
        rb, rkeep = packed(chd, ref, H, F.part(sel, B))
        sh = he.tick(rb, t * TICK, capi.TICK_ALL)
        assert_same(snapshot(fe, sf), snapshot(he, sh), "tick %d" % t)
        got, want = fe.get_query_status(H + B), he.get_query_status(H + B)
        assert (got[bad] == capi.Q_ERR_MISSING_ARRAY).all() and (want[bad] == capi.Q_ERR_BAD_STEP).all()
        keep_rows = np.setdiff1d(np.arange(H + B), bad)
        np.testing.assert_array_equal(got[keep_rows], want[keep_rows])
        check_follow(fe, F, status, want, H, sel)
    fe.close(), he.close()


@gpu
@pytest.mark.parametrize("adopted", [False, True], ids=["q", "adopted"])
def test_spot_buffer_grows_inside_one_size_class(chd, adopted):
    """Graphs on, the host part's size class fixed at 256: its spot total grows past the merged batch's spot buffer (4096 spots at
    first) while the follow stage replays from a graph, twice.  Every result and status equals the host-packed engine's."""
    capi, engine = chd.capi, chd.engine
    W = World(chd, 3000)
    S = 600
    lim = dict(max_pairs=1 << 17, max_queries=S + 512, max_spots=1 << 16)
    fe, he = W.engine(S, **lim), W.engine(S, **lim)
    for e in (fe, he):
        e.enable_graphs(True)
    slots = np.arange(0, S, 2, dtype=np.uint32)
    ent = W.rng.permutation(W.n)[:len(slots)]
    kind, shape = W.shapes(slots, True)
    W.follow(fe, slots, ent, kind, shape)
    F = Follow(W)
    F.bound(slots)
    B = len(slots)
    # spots per spot entry (3 of the 8 kinds carry spots): about 250 spots, then ~7 000 (> 4096), then ~20 000 (> 1.5 x 7 000)
    plan = [(1, 5), (1, 5), (1, 5), (80, 120), (80, 120), (80, 120), (240, 300), (240, 300)]
    grown = []
    for t, per in enumerate(plan, 1):
        if t > 1:
            W.step((fe, he), frac=0.3)
        n_h = 230 + 3 * t
        host = host_part(W, n_h, pick_slots(W.rng, n_h, S, W.bind), spots_per=per)
        H = engine.host_part_size(n_h)
        assert H == 256
        grown.append(int(host.spots[0][-1]))
        hb, hkeep = host.batch(engine)
        if adopted:
            fe.prefetch_queries(hb, hkeep)
            fe.adopt_prefetched()
            fe.follow_queries_with(capi.FOLLOW_MOVED, None)
        else:
            fe.follow_queries_with(capi.FOLLOW_MOVED, hb)
        sel, status = F.generate(1, {int(s) for s in host.sub if int(s) in W.bind})
        sf = fe.tick(None, t * TICK, capi.TICK_ALL | capi.TICK_FOLLOW)
        rb, rkeep = packed(chd, host, H, F.part(sel, B))
        sh = he.tick(rb, t * TICK, capi.TICK_ALL)
        assert_same(snapshot(fe, sf), snapshot(he, sh), "tick %d" % t)
        rs = he.get_query_status(H + B)
        np.testing.assert_array_equal(fe.get_query_status(H + B), rs)
        check_follow(fe, F, status, rs, H, sel)
    assert max(grown[:3]) < 4096 < min(grown[3:6]) and min(grown[6:]) > 1.5 * max(grown[3:6])
    assert fe.graph_launch_count() > 0
    fe.close(), he.close()


def result_set(torch, capi, S, Q, P):
    keep = dict(off=torch.zeros(S + 1, dtype=torch.int32).pin_memory(), ch=torch.zeros(P, dtype=torch.int32).pin_memory(),
                dist=torch.zeros(P, dtype=torch.int32).pin_memory(), new=[torch.zeros(P, dtype=torch.int32).pin_memory() for _ in range(4)],
                status=torch.zeros(Q, dtype=torch.int32).pin_memory(), voff=torch.zeros(S + 1, dtype=torch.int64).pin_memory(),
                hdr=torch.zeros(64, dtype=torch.int32).pin_memory())
    r = capi.ResultBuffers()
    r.pair_off, r.pair_channel, r.pair_dist, r.pair_cap = capi.ptr(keep["off"]), capi.ptr(keep["ch"]), capi.ptr(keep["dist"]), P
    r.new_sub, r.new_channel, r.unsub_sub, r.unsub_channel = (capi.ptr(t) for t in keep["new"])
    r.diff_cap = P
    r.query_status, r.status_cap, r.vis_off = capi.ptr(keep["status"]), Q, capi.ptr(keep["voff"])
    return r, keep


@gpu
def test_pipelined_loop_equals_serial(chd):
    """Host parts prefetched a tick ahead (both staging sets in use), adopted, merged, then CHD_TICK_FOLLOW + chd_fetch_results_async
    with the next tick enqueued before the wait: list by list the results of the serial form with the host part given directly.  One
    tick runs through chd_begin_interest."""
    capi, torch, engine = chd.capi, chd.torch, chd.engine
    W = World(chd, 20_000, cols=16, rows=16, table=True, seed=21)
    W.x, W.z = W.x.astype(np.float32).astype(np.float64), W.z.astype(np.float32).astype(np.float64)
    S = 3000
    P = 1 << 18
    lim = dict(max_pairs=P, max_visible=1 << 24, max_queries=S + 1024, max_spots=1 << 14)
    pe, se = W.engine(S, **lim), W.engine(S, **lim)
    slots = np.arange(0, S, 2, dtype=np.uint32)
    ent = W.rng.permutation(W.n)[:len(slots)]
    kind, shape = W.shapes(slots, True)
    for e in (pe, se):
        W.follow(e, slots, ent, kind, shape)
    T = 8
    moves, hosts = [], []
    for t in range(T):
        sel = W.rng.permutation(W.n)[:W.n // 10]
        moves.append((W.ids[sel].copy(), (W.x[sel] + W.rng.uniform(-30, 30, len(sel))).clip(0, 1599).astype(np.float32),
                      (W.z[sel] + W.rng.uniform(-30, 30, len(sel))).clip(0, 1599).astype(np.float32)))
        n_h = [120, 300, 90, 0, 260, 200, 40, 500][t]
        hosts.append(host_part(W, n_h, pick_slots(W.rng, n_h, S, W.bind)))
    Q = S + 1024
    serial = []
    for t, (mi, mx, mz) in enumerate(moves, 1):
        se.move_entities_f32(mi, mx, mz)
        hb, keep = hosts[t - 1].batch(engine)
        se.follow_queries_with(capi.FOLLOW_MOVED, hb)
        s = se.tick(None, t * TICK, capi.TICK_BUILD | capi.TICK_EMIT | capi.TICK_FOLLOW)
        p = se.get_pairs()
        (ns, nc), (us, uc) = se.get_diff(s.n_sub_new, s.n_unsub)
        n = engine.host_part_size(hosts[t - 1].n) + len(slots)
        serial.append(dict(summary=s.as_dict(), off=p["off"], ch=p["channel"], dist=p["dist"], new=sorted(zip(ns.tolist(), nc.tolist())),
                           unsub=sorted(zip(us.tolist(), uc.tolist())), status=se.get_query_status(n), voff=se.get_visible()[0],
                           follow=se.get_follow()))
    sets = [result_set(torch, capi, S, Q, P), result_set(torch, capi, S, Q, P)]

    def check(t, summ):
        want, (r, k) = serial[t], sets[t % 2]
        assert {f: getattr(summ, f) for f in want["summary"]} == want["summary"], t
        n = summ.n_pairs
        np.testing.assert_array_equal(k["off"].numpy().view(np.uint32), want["off"])
        np.testing.assert_array_equal(k["ch"].numpy().view(np.uint32)[:n], want["ch"])
        np.testing.assert_array_equal(k["dist"].numpy().view(np.uint32)[:n], want["dist"])
        nw = [a.numpy().view(np.uint32) for a in k["new"]]
        assert sorted(zip(nw[0][:summ.n_sub_new].tolist(), nw[1][:summ.n_sub_new].tolist())) == want["new"]
        assert sorted(zip(nw[2][:summ.n_unsub].tolist(), nw[3][:summ.n_unsub].tolist())) == want["unsub"]
        m = len(want["status"])
        np.testing.assert_array_equal(k["status"].numpy().view(np.uint32)[:m], want["status"])
        np.testing.assert_array_equal(k["voff"].numpy().view(np.uint64), want["voff"])

    summ = capi.TickSummary()
    keeps = [None, None]
    hb, keeps[0] = hosts[0].batch(engine)
    pe.prefetch_queries(hb, keeps[0])
    for t, (mi, mx, mz) in enumerate(moves):
        pe.move_entities_f32(mi, mx, mz)
        pe.adopt_prefetched()
        pe.follow_queries_with(capi.FOLLOW_MOVED, None)  # consumes the adopted host part: its staging set is free again
        if t + 1 < T:  # tick t + 1's host part goes into the other staging set while tick t runs
            hb, keeps[(t + 1) % 2] = hosts[t + 1].batch(engine)
            pe.prefetch_queries(hb, keeps[(t + 1) % 2])
        if t == 5:
            pe.begin_interest(None, (t + 1) * TICK, False)
            pe.tick(None, (t + 1) * TICK, capi.TICK_BUILD | capi.TICK_EMIT, want_summary=False)
        else:
            pe.tick(None, (t + 1) * TICK, capi.TICK_BUILD | capi.TICK_EMIT | capi.TICK_FOLLOW, want_summary=False)
        r, k = sets[t % 2]
        assert pe.L.chd_fetch_results_async(pe.h, C.byref(r), capi.ptr(k["hdr"])) == 0
        if t:
            assert pe.L.chd_fetch_wait(pe.h, C.byref(summ)) == 0
            check(t - 1, summ)
    assert pe.L.chd_fetch_wait(pe.h, C.byref(summ)) == 0
    check(T - 1, summ)
    f, want = pe.get_follow(), serial[-1]["follow"]
    for key in ("slot", "status", "cx", "cz"):
        np.testing.assert_array_equal(f[key], want[key])
    assert f["n_selected"] == want["n_selected"]
    pe.close(), se.close()


@gpu
def test_sizes_where_the_kernels_loop(chd):
    """Host parts of 0, 1, 255, 256, 257 and 2^17 + 1 entries on 600 K slots (the compaction spans more tiles than SMs) with up to
    max_queries - H followers (the merge's grid-stride loop runs several rounds), and a spot total that outgrows the spot buffer."""
    capi, engine, torch = chd.capi, chd.engine, chd.torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    S = 600_000
    assert (S + 4095) // 4096 > sms
    n_big = (1 << 17) + 1
    H_big = engine.host_part_size(n_big)
    B = 150_000
    Q = H_big + B
    assert Q > 4 * sms * 256  # the merge kernel's grid is at most 4 blocks of 256 per SM
    W = World(chd, 200_000, cols=64, rows=64, w=500.0, seed=13)
    lim = dict(max_pairs=6_000_000, max_visible=1 << 20, max_due=1 << 20, max_window_cells=16_000_000, max_queries=Q, max_spots=1 << 19)
    fe, he = W.engine(S, **lim), W.engine(S, **lim)
    slots = np.sort(W.rng.permutation(S)[:B]).astype(np.uint32)
    ent = W.rng.integers(0, W.n, B)
    kind, shape = W.shapes(slots, True)
    shape[0], shape[1], shape[2], shape[6] = 40.0, 30.0, 30.0, 60.0
    W.follow(fe, slots, ent, kind, shape)
    F = Follow(W)
    F.bound(slots)
    for t, n_h in enumerate([0, 1, 255, 256, 257, n_big, 3], 1):
        if t > 1:
            W.step((fe, he), frac=0.05)
        host = host_part(W, n_h, pick_slots(W.rng, n_h, S, W.bind), spots=True)
        if host.spots is not None and n_h == n_big:
            assert int(host.spots[0][-1]) > 4096 * 3 // 2  # more than the spot buffer the earlier ticks allocated
        H = engine.host_part_size(n_h)
        assert H + B <= Q
        hb, keep = host.batch(engine)
        fe.follow_queries_with(capi.FOLLOW_MOVED if t % 2 == 0 else capi.FOLLOW_ALL, hb)
        sel, status = F.generate(1 if t % 2 == 0 else 0, {int(s) for s in host.sub if int(s) in W.bind})
        sf = fe.tick(None, t * TICK, capi.TICK_BUILD | capi.TICK_FOLLOW)
        rb, rkeep = packed(chd, host, H, F.part(sel, B))
        sh = he.tick(rb, t * TICK, capi.TICK_BUILD)
        assert_same(snapshot(fe, sf, vis=False), snapshot(he, sh, vis=False), "tick %d" % t)
        rs = he.get_query_status(H + B)
        np.testing.assert_array_equal(fe.get_query_status(H + B), rs)
        check_follow(fe, F, status, rs, H, sel)
    # B up to max_queries - H: one more follower would not fit the largest class
    big, keep = host_part(W, n_big, pick_slots(W.rng, n_big, S, W.bind)).batch(engine)
    fe.follow_bind(np.array([int(np.setdiff1d(np.arange(S), slots)[0])], np.uint32), np.array([1], np.uint32), sph_r=np.array([10.0]))
    refused(fe, capi.ERR_CAPACITY, "max_queries", "chd_follow_queries_with", 0, C.byref(big))
    fe.close(), he.close()


@gpu
@pytest.mark.parametrize("table", [False, True], ids=["index", "table"])
def test_empty_host_part_is_bit_identical(chd, table):
    """n_h = 0 (an empty batch, and an adopted empty prefetch): the same launches as chd_follow_queries, and every result, status
    and follower report equal to its."""
    capi, engine = chd.capi, chd.engine
    W = World(chd, 3000, table=table)
    S = 500
    a, b = W.engine(S), W.engine(S)
    slots = np.arange(1, S, 2, dtype=np.uint32)
    ent = W.rng.permutation(W.n)[:len(slots)]
    kind, shape = W.shapes(slots, True)
    for e in (a, b):
        W.follow(e, slots, ent, kind, shape)
    B = len(slots)
    for t in range(1, 7):
        if t > 1:
            W.step((a, b), frac=0.4)
        mode = t % 2
        eb, keep = engine.make_batch(0, sub=np.zeros(0, np.uint32))
        if t % 3 == 0:
            b.prefetch_queries(eb, keep)
            b.adopt_prefetched()
        la, lb = a.launch_count(), b.launch_count()
        a.follow_queries(mode)
        b.follow_queries_with(mode, None if t % 3 == 0 else eb)
        assert a.launch_count() - la == b.launch_count() - lb
        sa = a.tick(None, t * TICK, capi.TICK_ALL | capi.TICK_FOLLOW)
        sb = b.tick(None, t * TICK, capi.TICK_ALL | capi.TICK_FOLLOW)
        assert_same(snapshot(a, sa), snapshot(b, sb), "tick %d" % t)
        np.testing.assert_array_equal(a.get_query_status(B), b.get_query_status(B))
        fa, fb = a.get_follow(), b.get_follow()
        for k in ("slot", "entity", "status", "cx", "cz"):
            np.testing.assert_array_equal(fa[k], fb[k])
        assert fa["n_selected"] == fb["n_selected"]
    assert a.graph_launch_count() == b.graph_launch_count()
    a.close(), b.close()


@gpu
def test_refusals_change_nothing(chd):
    """Every refusal of chd_follow_queries_with, each leaving the follower state and an adopted batch as they were; the existing
    calls keep their rules."""
    capi, engine = chd.capi, chd.engine
    W = World(chd, 800)
    S = 50
    fe, he = W.engine(S, max_queries=S + 256 + 64), W.engine(S, max_queries=S + 256 + 64)
    slots = np.arange(0, S, 2, dtype=np.uint32)
    ent = np.arange(len(slots)) * 3
    kind, shape = W.shapes(slots, True)
    W.follow(fe, slots, ent, kind, shape)
    F = Follow(W)
    F.bound(slots)
    B = len(slots)
    fe.follow_queries(capi.FOLLOW_ALL)
    fe.tick(None, TICK, capi.TICK_ALL | capi.TICK_FOLLOW)
    sel, _ = F.generate(0, set())
    rb, keep0 = packed(chd, host_part(W, 0, []), 0, F.part(sel, B))
    he.tick(rb, TICK, capi.TICK_ALL)
    before = fe.get_follow()
    host = host_part(W, 20, pick_slots(W.rng, 20, S, W.bind, unknown=False))
    hb, hkeep = host.batch(engine)
    ident, ikeep = engine.make_batch(3, sphere=(np.array([50.0] * 3), np.array([50.0] * 3), np.array([20.0] * 3)))
    q = C.byref(hb)
    # arguments
    refused(fe, capi.ERR_INVALID, None, "chd_follow_queries_with", 2, q)
    refused(fe, capi.ERR_INVALID, "identity batch", "chd_follow_queries_with", 0, C.byref(ident))
    assert fe.L.chd_follow_queries_with(None, 0, q) == capi.ERR_INVALID
    # capacity: H + B > max_queries (a class of 512 for 300 entries)
    wide = host_part(W, 300, np.arange(300) + S)
    wb, wkeep = wide.batch(engine)
    refused(fe, capi.ERR_CAPACITY, "max_queries", "chd_follow_queries_with", 0, C.byref(wb))
    # a generated batch pending; a chd_begin_interest pending
    fe.follow_queries(capi.FOLLOW_ALL)
    refused(fe, capi.ERR_STATE, "has not been consumed", "chd_follow_queries_with", 0, q)
    fe.begin_interest(None, 2 * TICK)
    refused(fe, capi.ERR_STATE, "pending", "chd_follow_queries_with", 0, q)
    fe.tick(None, 2 * TICK, capi.TICK_ALL)
    sel, _ = F.generate(0, set())
    rb, keep1 = packed(chd, host_part(W, 0, []), 0, F.part(sel, B))
    he.tick(rb, 2 * TICK, capi.TICK_ALL)
    # q == NULL without an adopted batch; q beside an adopted one; an adopted identity batch
    refused(fe, capi.ERR_STATE, "chd_adopt_prefetched", "chd_follow_queries_with", 0, None)
    fe.prefetch_queries(ident, ikeep)
    fe.adopt_prefetched()
    refused(fe, capi.ERR_STATE, "adopted", "chd_follow_queries_with", 0, q)
    refused(fe, capi.ERR_INVALID, "identity batch", "chd_follow_queries_with", 0, None)
    refused(fe, capi.ERR_STATE, "adopted prefetched", "chd_follow_queries", 0)  # (unchanged)
    # nothing changed: the follower report is the same, and the adopted batch still runs through chd_update_interest alone
    after = fe.get_follow()
    for k in ("slot", "entity", "status", "cx", "cz", "n_selected"):
        np.testing.assert_array_equal(after[k], before[k])
    fe.update_interest(None, 3 * TICK)
    he.update_interest(ident, 3 * TICK)
    np.testing.assert_array_equal(fe.get_query_status(3), he.get_query_status(3))
    for k in ("off", "channel", "dist"):
        np.testing.assert_array_equal(fe.get_pairs()[k], he.get_pairs()[k])
    # an adopted batch refused by the capacity check stays adopted
    fe.prefetch_queries(wb, wkeep)
    fe.adopt_prefetched()
    refused(fe, capi.ERR_CAPACITY, "max_queries", "chd_follow_queries_with", 0, None)
    fe.update_interest(None, 4 * TICK)
    he.update_interest(wb, 4 * TICK)
    np.testing.assert_array_equal(fe.get_query_status(300), he.get_query_status(300))
    # existing rules: chd_adopt_prefetched of queries while a merged (generated) batch is pending; a q with CHD_TICK_FOLLOW
    fe.follow_queries_with(capi.FOLLOW_ALL, hb)
    fe.prefetch_queries(ident, ikeep)
    refused(fe, capi.ERR_STATE, "one batch per update", "chd_adopt_prefetched")
    refused(fe, capi.ERR_INVALID, None, "chd_tick", q, 5 * TICK, capi.TICK_ALL | capi.TICK_FOLLOW, None)
    fe.tick(None, 5 * TICK, capi.TICK_ALL | capi.TICK_FOLLOW)
    # rule 9: a slab refuses the call
    slab = engine.Engine(W.cfg(), 10, 8)
    slab.set_subscribers(np.arange(1, 9, dtype=np.uint32))
    slab.set_slab(0, 4, 1)
    refused(slab, capi.ERR_STATE, "slab", "chd_follow_queries_with", 0, q)
    for e in (fe, he, slab):
        e.close()
