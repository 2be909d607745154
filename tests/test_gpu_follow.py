"""Followers (chd_follow_bind / chd_follow_queries): subscriber slots whose AOI is centred on an entity, the tick's query batch
generated on the device.  The reference for every check is the batch a host would have packed from its own position mirror, fed
to a second engine through the ordinary query path, and, for the sphere worlds, the CPU oracle.
Run on an H100:  python -m pytest tests -m gpu"""
import ctypes as C

import numpy as np
import pytest

gpu = pytest.mark.gpu
MS = 1_000_000
TICK = 33 * MS
SPHERE, BOX, CONE = 4, 2, 8


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


class World:
    """Positions as the host would mirror them (id -> x, z; index mode: id = index), and the follower bindings."""

    def __init__(self, chd, n, cols=8, rows=8, w=100.0, table=False, seed=3):
        self.chd, self.n, self.table = chd, n, table
        self.cols, self.rows, self.w = cols, rows, w
        rng = np.random.default_rng(seed)
        self.rng = rng
        self.x = rng.uniform(0, cols * w, n)
        self.z = rng.uniform(0, rows * w, n)
        self.ids = (np.arange(n, dtype=np.uint32) * 3 + 7) if table else np.arange(n, dtype=np.uint32)
        self.live = np.ones(n, bool)
        self.bind = {}  # slot -> (entity position index, kind, shape[7])

    def cfg(self):
        return self.chd.engine.grid_cfg(0, 0, self.w, self.w, self.cols, self.rows)

    def engine(self, n_slots, max_subs=None, **lim):
        e = self.chd.engine.Engine(self.cfg(), self.n + 16, max_subs or n_slots, **lim)  # (room for a few extra spawns)
        e.set_subscribers(np.arange(1, n_slots + 1, dtype=np.uint32))
        if self.table:
            e.entity_table_init()
            assert (e.spawn_entities(self.ids, self.x, self.z) == 0).all()
        else:
            e.set_entities(self.x, self.z)
        return e

    def shapes(self, slots, mix):
        m = len(slots)
        rng = self.rng
        kind = np.full(m, SPHERE, np.uint8)
        if mix:
            kind = np.array([SPHERE, BOX, CONE, SPHERE | BOX, SPHERE | CONE, BOX | CONE, SPHERE | BOX | CONE], np.uint8)[np.arange(m) % 7]
        ang = rng.uniform(0, 2 * np.pi, m)
        shape = np.stack([rng.uniform(20, 160, m), rng.uniform(10, 120, m), rng.uniform(10, 120, m), np.cos(ang), np.sin(ang),
                          rng.uniform(0.2, 1.4, m), rng.uniform(30, 180, m)])
        return kind, shape

    def follow(self, e, slots, ent, kind, shape):
        """binds on engine e (None: mirror only)"""
        for j, s in enumerate(slots):
            self.bind[int(s)] = (int(ent[j]), int(kind[j]), shape[:, j].copy())
        if e is not None:
            e.follow_bind(slots, self.ids[ent], kind=kind, sph_r=shape[0], box=(shape[1], shape[2]), cone=tuple(shape[3:7]))

    def pack(self, slots=None):
        """the batch a host packs for `slots` (default: every follower whose entity exists), ascending slot order"""
        sl = sorted(self.bind) if slots is None else sorted(int(s) for s in slots)
        sl = [s for s in sl if self.live[self.bind[s][0]]]
        m = len(sl)
        ent = np.array([self.bind[s][0] for s in sl], np.int64)
        kind = np.array([self.bind[s][1] for s in sl], np.uint8)
        sh = np.array([self.bind[s][2] for s in sl]).reshape(m, 7).T.copy()
        cx, cz = self.x[ent].copy(), self.z[ent].copy()
        return self.chd.engine.make_batch(m, sub=np.array(sl, np.uint32), kind=kind, sphere=(cx, cz, sh[0]), box=(cx, cz, sh[1], sh[2]),
                                          cone=(cx, cz, sh[3], sh[4], sh[5], sh[6]))

    def step(self, engines, frac=1.0, f32=False, step=35.0):
        """moves a fraction of the live entities inside the world, on the mirror and on every engine -> moved position indices"""
        idx = np.flatnonzero(self.live)
        if frac < 1.0:
            idx = self.rng.permutation(idx)[:max(1, int(len(idx) * frac))]
        nx = np.clip(self.x[idx] + self.rng.uniform(-step, step, len(idx)), 0, self.cols * self.w - 1e-3)
        nz = np.clip(self.z[idx] + self.rng.uniform(-step, step, len(idx)), 0, self.rows * self.w - 1e-3)
        if f32:
            nx, nz = nx.astype(np.float32).astype(np.float64), nz.astype(np.float32).astype(np.float64)
        self.x[idx], self.z[idx] = nx, nz
        for e in engines:
            if self.table:
                (e.move_entities_f32 if f32 else e.move_entities)(self.ids[idx], nx, nz)
            else:
                e.set_entities(self.x, self.z)
        return idx


def rings(chd, world, tick, n_conn, state):
    wc = chd.synth.WorldConfig("t", 0, 0, world.w, world.w, world.cols, world.rows, 1, 1, world.n, n_conn, 50.0, 11)
    return chd.synth.update_rings(wc, tick, tick * TICK, TICK, 3, n_conn, ring_len=16, state=state)


def snapshot(e, s, vis=True):
    """every host-facing result of the last tick, in a comparable form"""
    p = e.get_pairs()
    (ns, nc), (us, uc) = e.get_diff(s.n_sub_new, s.n_unsub)
    due = e.get_due(s.n_due)
    out = dict(summary=s.as_dict(), new=sorted(zip(ns.tolist(), nc.tolist())), unsub=sorted(zip(us.tolist(), uc.tolist())),
               due=sorted(map(tuple, due.tolist())))
    out.update({"pair_" + k: v for k, v in p.items()})
    if vis:
        out["vis_off"], out["vis"] = e.get_visible()
    return out


def assert_same(a, b, what=""):
    assert a.keys() == b.keys()
    for k in a:
        if isinstance(a[k], np.ndarray):
            np.testing.assert_array_equal(a[k], b[k], err_msg="%s %s" % (what, k))
        else:
            assert a[k] == b[k], (what, k)


@gpu
@pytest.mark.parametrize("table", [False, True], ids=["index", "table"])
@pytest.mark.parametrize("mix", [False, True], ids=["sphere", "mixed"])
@pytest.mark.parametrize("graphs", [True, False], ids=["graphs", "direct"])
def test_follow_equals_host_packed_batch(chd, table, mix, graphs):
    """12 ticks of moving entities with fan-out: a follow engine and an engine fed the host-packed batch agree on every result."""
    capi = chd.capi
    W = World(chd, 4000, table=table)
    S = 600
    fe, he = W.engine(S, max_pairs=1 << 16), W.engine(S, max_pairs=1 << 16)
    for e in (fe, he):
        e.enable_graphs(graphs)
    replays = 0
    slots = np.arange(0, S, 2, dtype=np.uint32)  # half of the slots follow; the others never query
    ent = W.rng.permutation(W.n)[:len(slots)]
    kind, shape = W.shapes(slots, mix)
    W.follow(fe, slots, ent, kind, shape)
    state = None
    for t in range(1, 13):
        if t > 1:
            W.step((fe, he), frac=0.5 if table else 1.0)
        state, off, arr, snd, idx, cmi = rings(chd, W, t, S, state)
        for e in (fe, he):
            e.set_rings(off, arr, snd, idx, cmi)
        g0 = fe.graph_launch_count()
        fe.follow_queries(capi.FOLLOW_ALL)
        replays += fe.graph_launch_count() - g0
        if t % 2:
            sf = fe.tick(None, t * TICK, capi.TICK_ALL | capi.TICK_FOLLOW)
        else:  # the same through the early start
            fe.begin_interest(None, t * TICK)
            sf = fe.tick(None, t * TICK, capi.TICK_ALL)
        batch, keep = W.pack()
        sh = he.tick(batch, t * TICK, capi.TICK_ALL)
        assert_same(snapshot(fe, sf), snapshot(he, sh), "tick %d" % t)
        np.testing.assert_array_equal(fe.get_query_status(len(slots)), he.get_query_status(len(slots)))
        f = fe.get_follow()
        np.testing.assert_array_equal(f["slot"], slots)
        np.testing.assert_array_equal(f["entity"], W.ids[ent])
        np.testing.assert_array_equal(f["cx"], W.x[ent])
        np.testing.assert_array_equal(f["cz"], W.z[ent])
        assert f["n_selected"] == len(slots) and (f["status"] == 0).all()
    assert sf.n_due > 0 and sf.n_kept > 0
    # the follow stage runs direct once, is captured at its second execution and replays from then on
    assert replays == (11 if graphs else 0), replays
    fe.close(), he.close()


@gpu
def test_follow_against_the_oracle(chd, oracle):
    """Sphere followers in index mode: pairs, visible lists and the interest diff equal the CPU oracle's on the mirror positions."""
    from tests._oracle import make_grid

    capi = chd.capi
    W = World(chd, 3000)
    S = 300
    fe = W.engine(S)
    slots = np.arange(S, dtype=np.uint32)
    ent = W.rng.permutation(W.n)[:S]
    kind, shape = W.shapes(slots, False)
    W.follow(fe, slots, ent, kind, shape)
    g = make_grid(0, 0, W.w, W.w, W.cols, W.rows)
    prev = None
    for t in range(1, 5):
        if t > 1:
            W.step((fe,))
        fe.follow_queries(capi.FOLLOW_ALL)
        s = fe.tick(None, t * TICK, capi.TICK_BUILD | capi.TICK_EMIT | capi.TICK_FOLLOW)
        want = oracle.sphere_tick(g, W.x, W.z, W.x[ent], W.z[ent], shape[0])
        assert (want["status"] == 0).all()
        p = fe.get_pairs()
        np.testing.assert_array_equal(p["off"], want["pair_off"].astype(np.uint32))
        np.testing.assert_array_equal(p["channel"], want["pair_cell"])
        np.testing.assert_array_equal(p["dist"], want["pair_dist"])
        voff, vis = fe.get_visible()
        np.testing.assert_array_equal(voff, want["vis_off"])
        np.testing.assert_array_equal(vis, want["vis_entity"])
        (ns, nc), (us, uc) = fe.get_diff(s.n_sub_new, s.n_unsub)
        new, gone = set(zip(ns.tolist(), nc.tolist())), set(zip(us.tolist(), uc.tolist()))
        wn, wg = set(), set()
        for sl in range(S):
            ex = prev["channel"][prev["off"][sl]:prev["off"][sl + 1]] if prev else np.zeros(0, np.uint32)
            un, sn, _ = oracle.interest_diff(ex, p["channel"][p["off"][sl]:p["off"][sl + 1]])
            wn |= {(sl, int(c)) for c in sn}
            wg |= {(sl, int(c)) for c in un}
        assert new == wn and gone == wg
        prev = p
    fe.close()


def winners(ids, x, z):
    """last move of each id in array order -> dict id -> (x, z)"""
    out = {}
    for i, a, b in zip(ids.tolist(), x.tolist(), z.tolist()):
        out[i] = (a, b)
    return out


@gpu
def test_moved_selects_exactly_the_movers(chd):
    """Table mode, 400 K ids, 160 K followers, 1 % moved per tick (f32 moves): CHD_FOLLOW_MOVED selects the followers whose entity's
    winning position changed bitwise, plus re-bound slots; the state equals that of an engine fed queries for those slots only."""
    capi = chd.capi
    N, S = 400_000, 160_000
    W = World(chd, N, cols=64, rows=64, w=500.0, table=True, seed=5)
    W.x, W.z = W.x.astype(np.float32).astype(np.float64), W.z.astype(np.float32).astype(np.float64)
    fe, he = W.engine(S), W.engine(S)
    slots = np.arange(S, dtype=np.uint32)
    ent = W.rng.permutation(N)[:S]
    kind, shape = W.shapes(slots, False)
    shape[0] = 60.0
    W.follow(fe, slots, ent, kind, shape)
    slot_of_ent = {int(p): int(s) for s, p in zip(slots, ent)}
    pos_of_id = {int(i): k for k, i in enumerate(W.ids)}
    flags = capi.TICK_BUILD | capi.TICK_FANOUT
    for t in range(1, 6):
        expect = set(slots.tolist()) if t == 1 else set()
        if t > 1:
            m = N // 100
            sel = W.rng.permutation(N)[:m]
            mid = W.ids[sel].copy()
            mx = np.clip(W.x[sel] + W.rng.uniform(-90, 90, m), 0, 31999).astype(np.float32)
            mz = np.clip(W.z[sel] + W.rng.uniform(-90, 90, m), 0, 31999).astype(np.float32)
            fol = W.rng.permutation(ent)[:6]
            # a move to the position it already has; two moves of one id (the last wins); a move of an unknown id
            mid = np.concatenate([mid, W.ids[fol[:4]], [W.ids[fol[2]], 2, W.ids[fol[4]]]]).astype(np.uint32)
            mx = np.concatenate([mx, [W.x[fol[0]], W.x[fol[1]] + 8, 100.0, W.x[fol[3]]], [W.x[fol[2]] + 16, 5.0, W.x[fol[4]] + 4]]).astype(np.float32)
            mz = np.concatenate([mz, [W.z[fol[0]], W.z[fol[1]], 100.0, W.z[fol[3]] + 8], [W.z[fol[2]], 5.0, W.z[fol[4]]]]).astype(np.float32)
            for e in (fe, he):
                e.move_entities_f32(mid, mx, mz)
            for i, (a, b) in winners(mid, mx.astype(np.float64), mz.astype(np.float64)).items():
                k = pos_of_id.get(i)
                if k is None:
                    continue
                if (a != W.x[k] or b != W.z[k]) and k in slot_of_ent:
                    expect.add(slot_of_ent[k])
                W.x[k], W.z[k] = a, b
            assert slot_of_ent[int(fol[0])] not in expect or int(fol[0]) in sel
            if t == 3:  # a re-bound slot is selected although its entity stood still
                rb = np.array([s for s in range(S) if s not in expect][:3], np.uint32)
                re = np.array([W.bind[int(s)][0] for s in rb])
                W.follow(fe, rb, re, np.full(3, SPHERE, np.uint8), np.tile(np.array([[75.0], [0], [0], [0], [0], [0], [0]]), (1, 3)))
                expect |= set(rb.tolist())
        fe.follow_queries(capi.FOLLOW_MOVED)
        sf = fe.tick(None, t * TICK, flags | capi.TICK_FOLLOW)
        batch, keep = W.pack(sorted(expect))
        sh = he.tick(batch, t * TICK, flags)
        f = fe.get_follow()
        got = f["slot"][f["status"] != capi.FOLLOW_NOT_SELECTED]
        np.testing.assert_array_equal(got, np.array(sorted(expect), np.uint32))
        assert f["n_selected"] == len(expect) and (f["status"][f["status"] != capi.FOLLOW_NOT_SELECTED] == 0).all()
        np.testing.assert_array_equal(f["cx"], W.x[ent])
        assert_same(snapshot(fe, sf, vis=False), snapshot(he, sh, vis=False), "tick %d" % t)
    st = fe.entity_stats()
    assert st["moves_unknown"] == 4 and st["moves_superseded"] >= 4
    fe.close(), he.close()


@gpu
@pytest.mark.parametrize("B", [0, 1, 4095, 4096, 4097])
def test_follow_batch_sizes_around_one_tile(chd, B):
    capi = chd.capi
    W = World(chd, 6000)
    S = 4200
    fe, he = W.engine(S, max_pairs=1 << 18), W.engine(S, max_pairs=1 << 18)
    slots = np.arange(B, dtype=np.uint32)
    ent = W.rng.integers(0, W.n, B)
    kind, shape = W.shapes(slots, True)
    if B:
        W.follow(fe, slots, ent, kind, shape)
    for t in (1, 2):
        if t == 2:
            W.step((fe, he))
        fe.follow_queries(capi.FOLLOW_ALL)
        sf = fe.tick(None, t * TICK, capi.TICK_BUILD | capi.TICK_FOLLOW)
        batch, keep = W.pack()
        sh = he.tick(batch, t * TICK, capi.TICK_BUILD)
        assert_same(snapshot(fe, sf, vis=False), snapshot(he, sh, vis=False))
        assert fe.get_follow()["n_selected"] == B
    fe.close(), he.close()


@gpu
def test_follow_generation_spans_more_tiles_than_sms(chd):
    """1.2 M slots, every 7th one a follower (slot order != dense order): the compaction's look-back runs over more tiles than the
    device has SMs, and the selected list, centres and resulting subscriptions equal the host-packed engine's."""
    capi = chd.capi
    S = 1_200_000
    sms = chd.torch.cuda.get_device_properties(0).multi_processor_count
    assert (S + 4095) // 4096 > sms
    W = World(chd, 200_000, cols=64, rows=64, w=500.0, table=True, seed=9)
    lim = dict(max_pairs=4_000_000, max_visible=1 << 20, max_due=1 << 20, max_window_cells=8_000_000)
    fe, he = W.engine(S, **lim), W.engine(S, **lim)
    slots = np.arange(3, S, 7, dtype=np.uint32)
    ent = W.rng.integers(0, W.n, len(slots))
    kind, shape = W.shapes(slots, True)
    W.follow(fe, slots, ent, kind, shape)
    for t, mode in ((1, capi.FOLLOW_ALL), (2, capi.FOLLOW_MOVED), (3, capi.FOLLOW_ALL)):
        moved = set(W.step((fe, he), frac=0.05).tolist()) if t > 1 else set()
        fe.follow_queries(mode)
        sf = fe.tick(None, t * TICK, capi.TICK_BUILD | capi.TICK_FOLLOW)
        sel = slots if mode == capi.FOLLOW_ALL else np.array([s for s, p in zip(slots, ent) if int(p) in moved], np.uint32)
        batch, keep = W.pack(sel)
        sh = he.tick(batch, t * TICK, capi.TICK_BUILD)
        f = fe.get_follow()
        np.testing.assert_array_equal(f["slot"], slots)
        np.testing.assert_array_equal(f["slot"][f["status"] == 0], sel)
        np.testing.assert_array_equal(f["cx"], W.x[ent])
        np.testing.assert_array_equal(f["cz"], W.z[ent])
        assert f["n_selected"] == len(sel)
        assert_same(snapshot(fe, sf, vis=False), snapshot(he, sh, vis=False), "tick %d" % t)
    fe.close(), he.close()


@gpu
def test_missing_and_out_of_world_entities(chd):
    capi = chd.capi
    W = World(chd, 500, table=True)
    S = 40
    fe = W.engine(S)
    slots = np.arange(S, dtype=np.uint32)
    ent = np.arange(S)
    kind, shape = W.shapes(slots, False)
    W.follow(fe, slots, ent, kind, shape)

    def tick(t, mode):
        fe.follow_queries(mode)
        s = fe.tick(None, t * TICK, capi.TICK_ALL | capi.TICK_FOLLOW)
        return s, fe.get_follow(), fe.get_pairs()

    s, f, p0 = tick(1, capi.FOLLOW_ALL)
    assert (f["status"] == 0).all() and s.n_pairs > 0
    # despawn the entity of slot 5, and spawn another id: it takes the freed table slot and must not be followed
    assert (fe.despawn_entities(W.ids[5:6]) == 0).all()
    assert (fe.spawn_entities(np.array([999_999], np.uint32), np.array([11.0]), np.array([12.0])) == 0).all()
    for t, mode in ((2, capi.FOLLOW_ALL), (3, capi.FOLLOW_MOVED)):
        s, f, p = tick(t, mode)
        assert f["status"][5] == capi.FOLLOW_NO_ENTITY and s.n_unsub == 0 and s.n_query_errors == 0
        assert f["n_selected"] == (S - 1 if mode == capi.FOLLOW_ALL else 0)
        for k in ("off", "channel", "dist", "interval"):
            np.testing.assert_array_equal(p[k], p0[k])
    # the id comes back (in another table slot): the follower resumes and counts as moved
    assert (fe.spawn_entities(W.ids[5:6], W.x[5:6], W.z[5:6]) == 0).all()
    s, f, p = tick(4, capi.FOLLOW_MOVED)
    assert f["n_selected"] == 1 and f["status"][5] == 0 and f["cx"][5] == W.x[5]
    np.testing.assert_array_equal(p["channel"], p0["channel"])
    # an entity moved out of the world: its query fails like any query centred out of the world
    fe.move_entities(W.ids[7:8], np.array([-50.0]), np.array([10.0]))
    s, f, p = tick(5, capi.FOLLOW_MOVED)
    assert f["status"][7] == capi.Q_ERR_OUT_OF_WORLD and s.n_query_errors == 1 and s.n_unsub == 0 and f["n_selected"] == 1
    np.testing.assert_array_equal(p["channel"], p0["channel"])
    fe.close()
    # index mode: an entity index at or above the entity count
    W = World(chd, 100)
    fe = W.engine(4)
    fe.follow_bind(np.array([0, 1], np.uint32), np.array([5, 100], np.uint32), sph_r=np.array([50.0, 50.0]))
    fe.follow_queries(capi.FOLLOW_ALL)
    fe.tick(None, TICK, capi.TICK_ALL | capi.TICK_FOLLOW)
    f = fe.get_follow()
    assert f["status"].tolist() == [0, capi.FOLLOW_NO_ENTITY] and f["n_selected"] == 1
    fe.close()


def refused(e, status, text, fn, *args):
    L = e.L
    st = getattr(L, fn)(e.h, *args)
    assert st == status, (fn, st)
    if text:
        assert text in L.chd_last_error(e.h).decode(), L.chd_last_error(e.h)


@gpu
def test_lifecycle_and_rules(chd):
    capi, engine = chd.capi, chd.engine
    W = World(chd, 800)
    S = 50
    fe, he = W.engine(S, max_subs=64), W.engine(S, max_subs=64)
    slots = np.arange(S, dtype=np.uint32)
    ent = np.arange(S) * 3
    kind, shape = W.shapes(slots, True)
    W.follow(fe, slots, ent, kind, shape)

    def both(t, mode=capi.FOLLOW_ALL, pack=None):
        fe.follow_queries(mode)
        sf = fe.tick(None, t * TICK, capi.TICK_ALL | capi.TICK_FOLLOW)
        batch, keep = W.pack(pack)
        sh = he.tick(batch, t * TICK, capi.TICK_ALL)
        assert_same(snapshot(fe, sf), snapshot(he, sh), "tick %d" % t)
        return sf

    both(1)
    # a removed follower: its pairs are in that update's unsub list, and it is not selected afterwards
    for e in (fe, he):
        e.remove_subscribers(np.array([4], np.uint32))
    del W.bind[4]
    s = both(2)
    (_, _), (us, _) = fe.get_diff(s.n_sub_new, s.n_unsub)
    assert s.n_unsub > 0 and set(us.tolist()) == {4}
    assert 4 not in fe.get_follow()["slot"]
    # unbind keeps the subscriptions
    fe.follow_unbind(np.array([6, 7], np.uint32))
    del W.bind[6], W.bind[7]
    W.step((fe, he))
    s = both(3)
    p = fe.get_pairs()
    assert p["off"][7] > p["off"][6] and not {6, 7} & set(fe.get_follow()["slot"].tolist())
    # argument checks: nothing is bound by a refused call
    one = np.array([1], np.uint32)
    r = np.array([10.0])

    def fb(slot=one, entity=one, kind=None, **kw):
        b = capi.FollowBatch()
        keep = [np.ascontiguousarray(slot, np.uint32), np.ascontiguousarray(entity, np.uint32)]
        b.n, b.slot, b.entity = len(keep[0]), capi.ptr(keep[0]), capi.ptr(keep[1])
        if kind is not None:
            keep.append(np.ascontiguousarray(kind, np.uint8))
            b.kind = capi.ptr(keep[-1])
        for k, v in kw.items():
            keep.append(np.ascontiguousarray(v, np.float64))
            setattr(b, k, capi.ptr(keep[-1]))
        b._keep = keep
        return C.byref(b)

    refused(fe, capi.ERR_INVALID, "never added", "chd_follow_bind", fb(slot=[60], sph_r=r))
    refused(fe, capi.ERR_INVALID, "never added", "chd_follow_bind", fb(slot=[64], sph_r=r))
    refused(fe, capi.ERR_INVALID, "CHD_AOI_SPOTS", "chd_follow_bind", fb(kind=[SPHERE | 1], sph_r=r))
    refused(fe, capi.ERR_INVALID, "not a mask", "chd_follow_bind", fb(kind=[0], sph_r=r))
    refused(fe, capi.ERR_INVALID, "is NULL", "chd_follow_bind", fb(kind=[BOX], sph_r=r))
    refused(fe, capi.ERR_INVALID, "is NULL", "chd_follow_bind", fb())
    refused(fe, capi.ERR_INVALID, None, "chd_follow_queries", 2)
    refused(fe, capi.ERR_INVALID, None, "chd_follow_unbind", capi.ptr(np.array([64], np.uint32)), 1)
    assert len(fe.get_follow()["slot"]) == len(W.bind)
    small = engine.Engine(W.cfg(), 10, 8, max_queries=2)
    small.set_subscribers(np.arange(1, 9, dtype=np.uint32))
    refused(small, capi.ERR_CAPACITY, "max_queries", "chd_follow_bind", fb(slot=[0, 1, 2], entity=[0, 1, 2], sph_r=[1.0, 1.0, 1.0]))
    refused(small, capi.OK, None, "chd_follow_bind", fb(slot=[0, 1, 1], entity=[0, 1, 2], sph_r=[1.0, 1.0, 1.0]))  # a slot twice: one follower
    # one batch per interest update
    batch, keep = W.pack()
    fe.follow_queries(capi.FOLLOW_ALL)
    refused(fe, capi.ERR_STATE, "has not been consumed", "chd_follow_queries", 0)
    fe.prefetch_queries(batch, keep)
    refused(fe, capi.ERR_STATE, "one batch per update", "chd_adopt_prefetched")
    refused(fe, capi.ERR_STATE, "has not been consumed", "chd_get_follow", None, None, None, None, None, 0, None, None)
    fe.update_interest(None, 4 * TICK)  # consumes the generated batch
    fe.adopt_prefetched()
    refused(fe, capi.ERR_STATE, "adopted prefetched", "chd_follow_queries", 0)
    fe.update_interest(None, 4 * TICK)
    refused(fe, capi.ERR_STATE, "CHD_TICK_FOLLOW without", "chd_tick", None, 5 * TICK, capi.TICK_ALL | capi.TICK_FOLLOW, None)
    fe.follow_queries(capi.FOLLOW_ALL)
    refused(fe, capi.ERR_INVALID, None, "chd_tick", C.byref(batch), 5 * TICK, capi.TICK_ALL | capi.TICK_FOLLOW, None)
    fe.begin_interest(None, 5 * TICK)
    refused(fe, capi.ERR_STATE, "pending", "chd_follow_queries", 0)
    fe.tick(None, 5 * TICK, capi.TICK_ALL)
    # rule 9: no followers on a slab, no slab on an engine with followers
    refused(fe, capi.ERR_STATE, "follow entities", "chd_set_slab", 0, 4, 1)
    refused(fe, capi.ERR_STATE, "follow entities", "chd_comm_init", (C.c_uint8 * 128)(), 0, 1, 1, 16, 0, 0)
    slab = engine.Engine(W.cfg(), 10, 8)
    slab.set_subscribers(np.arange(1, 9, dtype=np.uint32))
    slab.set_slab(0, 4, 1)
    refused(slab, capi.ERR_STATE, "slab", "chd_follow_bind", fb(sph_r=r))
    refused(slab, capi.ERR_STATE, "slab", "chd_follow_queries", 0)
    refused(slab, capi.ERR_STATE, "slab", "chd_follow_unbind", capi.ptr(one), 1)
    refused(slab, capi.ERR_STATE, "slab", "chd_get_follow", None, None, None, None, None, 0, None, None)
    # chd_set_subscribers clears every binding; an engine without followers generates an empty batch
    fe.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
    assert len(fe.get_follow()["slot"]) == 0
    fe.follow_queries(capi.FOLLOW_MOVED)
    s = fe.tick(None, 6 * TICK, capi.TICK_ALL | capi.TICK_FOLLOW)
    assert s.n_pairs == 0
    refused(fe, capi.OK, None, "chd_set_slab", 0, 4, 1)
    for e in (fe, he, small, slab):
        e.close()


@gpu
def test_pairs_overflow_on_a_moved_tick_is_repaired_by_an_all_tick(chd):
    capi = chd.capi
    W = World(chd, 2000)
    S = 200
    slots = np.arange(S, dtype=np.uint32)
    ent = np.arange(S) * 5
    kind, shape = W.shapes(slots, False)
    shape[0] = 40.0
    probe = W.engine(S)
    W.follow(probe, slots, ent, kind, shape)
    probe.follow_queries(capi.FOLLOW_ALL)
    n0 = probe.tick(None, TICK, capi.TICK_BUILD | capi.TICK_FOLLOW).n_pairs
    probe.close()
    W.bind.clear()
    fe, he = W.engine(S, max_pairs=n0 + n0 // 2), W.engine(S, max_pairs=1 << 16)
    W.follow(fe, slots, ent, kind, shape)
    fe.follow_queries(capi.FOLLOW_ALL)
    assert fe.tick(None, TICK, capi.TICK_BUILD | capi.TICK_FOLLOW).n_pairs == n0
    # entities move and half of the slots get wider shapes: the MOVED tick overflows the pair capacity and applies nothing, but the
    # movers' stored centres have advanced
    W.step((fe, he), frac=0.3)
    wide = slots[::2]
    big = shape[:, ::2].copy()
    big[0] = 260.0
    W.follow(fe, wide, ent[::2], kind[::2], big)
    fe.follow_queries(capi.FOLLOW_MOVED)
    with pytest.raises(capi.ChdError):
        fe.tick(None, 2 * TICK, capi.TICK_BUILD | capi.TICK_FOLLOW)
    assert fe.summary().n_pairs == n0
    # back to shapes that fit; MOVED would now skip the movers that were not re-bound, ALL repairs them
    W.follow(fe, wide, ent[::2], kind[::2], shape[:, ::2].copy() * 1.5)
    fe.follow_queries(capi.FOLLOW_ALL)
    sf = fe.tick(None, 3 * TICK, capi.TICK_BUILD | capi.TICK_FOLLOW)
    batch, keep = W.pack()
    he.tick(batch, 3 * TICK, capi.TICK_BUILD)
    pf, ph = fe.get_pairs(), he.get_pairs()
    for k in ("off", "channel", "dist", "interval"):
        np.testing.assert_array_equal(pf[k], ph[k])
    assert sf.overflow == 0
    fe.close(), he.close()


@gpu
def test_pipelined_loop_equals_serial(chd):
    """move_entities_f32 -> follow_queries -> begin_interest(NULL) -> tick -> fetch_results_async with the next tick enqueued before
    the wait: list by list the results of the serial form (the generation of tick k + 1 does not disturb tick k's batch)."""
    capi, torch = chd.capi, chd.torch
    W = World(chd, 20_000, cols=16, rows=16, table=True, seed=21)
    W.x, W.z = W.x.astype(np.float32).astype(np.float64), W.z.astype(np.float32).astype(np.float64)
    S = 3000
    lim = dict(max_pairs=1 << 18, max_visible=1 << 24)
    pe, se = W.engine(S, **lim), W.engine(S, **lim)
    slots = np.arange(S, dtype=np.uint32)
    ent = W.rng.permutation(W.n)[:S]
    kind, shape = W.shapes(slots, True)
    for e in (pe, se):
        W.follow(e, slots, ent, kind, shape)
    L = pe.L
    P = 1 << 18

    def result_set():
        keep = dict(off=torch.zeros(S + 1, dtype=torch.int32).pin_memory(), ch=torch.zeros(P, dtype=torch.int32).pin_memory(),
                    dist=torch.zeros(P, dtype=torch.int32).pin_memory(), new=[torch.zeros(P, dtype=torch.int32).pin_memory() for _ in range(4)],
                    status=torch.zeros(S, dtype=torch.int32).pin_memory(), voff=torch.zeros(S + 1, dtype=torch.int64).pin_memory(),
                    hdr=torch.zeros(64, dtype=torch.int32).pin_memory())
        r = capi.ResultBuffers()
        r.pair_off, r.pair_channel, r.pair_dist, r.pair_cap = capi.ptr(keep["off"]), capi.ptr(keep["ch"]), capi.ptr(keep["dist"]), P
        r.new_sub, r.new_channel, r.unsub_sub, r.unsub_channel = (capi.ptr(t) for t in keep["new"])
        r.diff_cap = P
        r.query_status, r.status_cap, r.vis_off = capi.ptr(keep["status"]), S, capi.ptr(keep["voff"])
        return r, keep

    sets = [result_set(), result_set()]
    moves = []
    for t in range(8):
        sel = W.rng.permutation(W.n)[:W.n // 10]
        moves.append((W.ids[sel].copy(), (W.x[sel] + W.rng.uniform(-30, 30, len(sel))).clip(0, 1599).astype(np.float32),
                      (W.z[sel] + W.rng.uniform(-30, 30, len(sel))).clip(0, 1599).astype(np.float32)))
    serial = []
    for t, (mi, mx, mz) in enumerate(moves, 1):
        se.move_entities_f32(mi, mx, mz)
        se.follow_queries(capi.FOLLOW_MOVED)
        se.begin_interest(None, t * TICK, False)
        s = se.tick(None, t * TICK, capi.TICK_BUILD | capi.TICK_EMIT)
        p = se.get_pairs()
        (ns, nc), (us, uc) = se.get_diff(s.n_sub_new, s.n_unsub)
        serial.append(dict(summary=s.as_dict(), off=p["off"], ch=p["channel"], dist=p["dist"], new=sorted(zip(ns.tolist(), nc.tolist())),
                           unsub=sorted(zip(us.tolist(), uc.tolist())), status=se.get_query_status(S), voff=se.get_visible()[0]))

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
        np.testing.assert_array_equal(k["status"].numpy().view(np.uint32), want["status"])
        np.testing.assert_array_equal(k["voff"].numpy().view(np.uint64), want["voff"])

    summ = capi.TickSummary()
    for t, (mi, mx, mz) in enumerate(moves):
        pe.move_entities_f32(mi, mx, mz)
        pe.follow_queries(capi.FOLLOW_MOVED)
        pe.begin_interest(None, (t + 1) * TICK, False)
        pe.tick(None, (t + 1) * TICK, capi.TICK_BUILD | capi.TICK_EMIT, want_summary=False)
        r, k = sets[t % 2]
        assert L.chd_fetch_results_async(pe.h, C.byref(r), capi.ptr(k["hdr"])) == 0
        if t:
            assert L.chd_fetch_wait(pe.h, C.byref(summ)) == 0
            check(t - 1, summ)
    assert L.chd_fetch_wait(pe.h, C.byref(summ)) == 0
    check(7, summ)
    pe.close(), se.close()
