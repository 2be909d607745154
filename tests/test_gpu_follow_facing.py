"""Followers that turn with their entity (include/chd_gpu_facing.h): facings carried by entity events, follower frames, and the
offset centres and cone directions generated from them on the device.  The reference is the one of tests/test_gpu_follow.py: the
batch a host would pack from its own mirror, here with the centres and directions restated in numpy in the header's operation order
(tests/_facing.py), fed to a second engine through the ordinary query path.
Run on an H100:  python -m pytest tests/test_gpu_follow_facing.py -m gpu"""
import ctypes as C

import numpy as np
import pytest

from tests._facing import frame_query
from tests.test_gpu_follow import assert_same, refused, rings, snapshot
from tests.test_gpu_sharded_follow import COLS, ROWS, W, Slabs, Walk, _bind, _cfg, _outside, _results, _shapes, _summary_fields
from tests.test_gpu_sharded_table import _vis_sets

pytestmark = pytest.mark.gpu

MS = 1_000_000
TICK = 33 * MS
SPHERE, BOX, CONE = 4, 2, 8
KINDS = np.array([CONE, SPHERE | CONE, BOX | CONE, SPHERE, BOX, SPHERE | BOX | CONE, SPHERE | BOX], np.uint8)


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
    ns.capi, ns.engine, ns.sharding, ns.synth, ns.torch = capi, engine, sharding, synth, torch
    return ns


def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


class FWorld:
    """The host's view of a table-mode world with facings: positions, facings and the followers' bindings and frames, and what the
    device's generation must have done (last inputs, dirty marks, the last framed queries)."""

    def __init__(self, chd, n, cols=16, rows=16, w=100.0, seed=3):
        self.chd, self.n, self.cols, self.rows, self.w = chd, n, cols, rows, w
        self.rng = rng = np.random.default_rng(seed)
        self.ids = np.arange(n, dtype=np.uint32) * 3 + 7
        self.x, self.z = rng.uniform(0, cols * w, n), rng.uniform(0, rows * w, n)
        yaw = rng.uniform(0, 2 * np.pi, n)
        self.fx, self.fz = np.cos(yaw), np.sin(yaw)
        self.fx[::17] = self.fz[::17] = 0.0  # entities without a facing
        self.live = np.ones(n, bool)
        self.bind, self.frame = {}, {}  # slot -> (entity index, kind, shape[7]) / (off_fwd, off_right, rot_cos, rot_sin)
        self.last, self.dirty, self.gen = {}, set(), {}  # slot -> inputs of its last query / dirty slots / framed: (fx, fz, cx, cz, dx, dz)

    def cfg(self):
        return self.chd.engine.grid_cfg(0, 0, self.w, self.w, self.cols, self.rows)

    def engine(self, n_slots, facing, **lim):
        e = self.chd.engine.Engine(self.cfg(), self.n + 64, n_slots, **lim)
        e.set_subscribers(np.arange(1, n_slots + 1, dtype=np.uint32))
        e.entity_table_init()
        if facing:
            assert (e.spawn_entities_facing(self.ids, self.x, self.z, self.fx, self.fz) == 0).all()
        else:
            assert (e.spawn_entities(self.ids, self.x, self.z) == 0).all()
        return e

    def shapes(self, m):
        rng = self.rng
        kind = KINDS[np.arange(m) % len(KINDS)]
        ang = rng.uniform(0, 2 * np.pi, m)
        return kind, np.stack([rng.uniform(20, 160, m), rng.uniform(10, 120, m), rng.uniform(10, 120, m), np.cos(ang), np.sin(ang),
                               rng.uniform(0.2, 1.4, m), rng.uniform(30, 180, m)])

    def follow(self, e, slots, ent, kind, shape):
        for j, s in enumerate(slots):
            s = int(s)
            self.bind[s] = (int(ent[j]), int(kind[j]), shape[:, j].copy())
            self.frame.pop(s, None)
            self.gen.pop(s, None)
            self.dirty.add(s)
        if e is not None:
            e.follow_bind(slots, self.ids[ent], kind=kind, sph_r=shape[0], box=(shape[1], shape[2]), cone=tuple(shape[3:7]))

    def set_frame(self, e, slots, fwd, right, rot=None):
        m = len(slots)
        fwd, right = np.broadcast_to(np.asarray(fwd, np.float64), (m,)), np.broadcast_to(np.asarray(right, np.float64), (m,))
        rc, rs = (np.ones(m), np.zeros(m)) if rot is None else (np.broadcast_to(rot[0], (m,)), np.broadcast_to(rot[1], (m,)))
        for j, s in enumerate(slots):
            s = int(s)
            self.frame[s] = (float(fwd[j]), float(right[j]), float(rc[j]), float(rs[j]))
            self.gen[s] = (0.0,) * 6
            self.dirty.add(s)
        if e is not None:
            e.follow_set_frame(slots, fwd, right, rot)

    def unframe(self, slots):
        for s in slots:
            self.frame.pop(int(s), None)
            self.gen.pop(int(s), None)

    def queries(self, slots):
        """-> [6][m]: (fx, fz, cx, cz, dx, dz) of each slot's query now (plain: no facing, the entity's position, the bound direction)"""
        m = len(slots)
        k = np.array([self.bind[s][0] for s in slots], np.int64)
        sh = np.array([self.bind[s][2] for s in slots]).reshape(m, 7)
        fr = np.array([self.frame.get(s, (0.0, 0.0, 1.0, 0.0)) for s in slots]).reshape(m, 4)
        framed = np.array([s in self.frame for s in slots], bool)
        q = np.array(frame_query(self.x[k], self.z[k], self.fx[k], self.fz[k], fr[:, 0], fr[:, 1], fr[:, 2], fr[:, 3], sh[:, 3], sh[:, 4])).reshape(6, m)
        q[0:2, ~framed] = 0.0
        q[2, ~framed], q[3, ~framed] = self.x[k[~framed]], self.z[k[~framed]]
        q[4, ~framed], q[5, ~framed] = sh[~framed, 3], sh[~framed, 4]
        return q, k, framed

    def select(self, mode):
        """the slots the generation selects (in slot order), applying the selection to the expectations"""
        capi = self.chd.capi
        slots = [s for s in sorted(self.bind) if self.live[self.bind[s][0]]]
        for s in sorted(self.bind):
            if not self.live[self.bind[s][0]]:
                self.dirty.add(s)
        if not slots:
            return []
        q, k, framed = self.queries(slots)
        kx, kz, kfx, kfz = bits(self.x[k]), bits(self.z[k]), bits(q[0]), bits(q[1])
        sel = []
        for j, s in enumerate(slots):
            key = (int(kx[j]), int(kz[j])) + ((int(kfx[j]), int(kfz[j])) if framed[j] else ())
            if mode == capi.FOLLOW_ALL or s in self.dirty or self.last.get(s) != key:
                sel.append(s)
                self.last[s] = key
                self.dirty.discard(s)
                if framed[j]:
                    self.gen[s] = tuple(float(v) for v in q[:, j])
        return sel

    def pack(self, sel):
        m = len(sel)
        q = self.queries(sel)[0] if m else np.zeros((6, 0))
        sh = np.array([self.bind[s][2] for s in sel]).reshape(m, 7).T.copy()
        kind = np.array([self.bind[s][1] for s in sel], np.uint8)
        cx, cz = q[2].copy(), q[3].copy()
        return self.chd.engine.make_batch(m, sub=np.array(sel, np.uint32), kind=kind, sphere=(cx, cz, sh[0]), box=(cx, cz, sh[1], sh[2]),
                                          cone=(cx, cz, q[4].copy(), q[5].copy(), sh[5], sh[6]))

    def apply(self, e):
        """binds and frames every follower of the mirror on e"""
        slots = np.array(sorted(self.bind), np.uint32)
        ent = np.array([self.bind[int(s)][0] for s in slots], np.int64)
        kind = np.array([self.bind[int(s)][1] for s in slots], np.uint8)
        sh = np.array([self.bind[int(s)][2] for s in slots]).reshape(len(slots), 7).T.copy()
        e.follow_bind(slots, self.ids[ent], kind=kind, sph_r=sh[0], box=(sh[1], sh[2]), cone=tuple(sh[3:7]))
        fs = np.array(sorted(self.frame), np.uint32)
        fr = np.array([self.frame[int(s)] for s in fs]).reshape(len(fs), 4).T.copy()
        e.follow_set_frame(fs, fr[0], fr[1], (fr[2], fr[3]))

    def events(self, fe, he, plain=None, facing=None, f32=False):
        """plain = (idx, x, z) moves without a facing, then facing = (idx, x, z, fx, fz) moves with one, on the mirror and both engines
        (he gets the positions only); each list may name an index twice (the last wins)"""
        cast = (lambda a: np.asarray(a, np.float32)) if f32 else (lambda a: np.asarray(a, np.float64))
        for ev, has in ((plain, False), (facing, True)):
            if ev is None or not len(ev[0]):
                continue
            idx = np.asarray(ev[0])
            vals = [cast(a) for a in ev[1:]]
            for j, k in enumerate(idx.tolist()):
                self.x[k], self.z[k] = float(vals[0][j]), float(vals[1][j])
                if has:
                    self.fx[k], self.fz[k] = float(vals[2][j]), float(vals[3][j])
            ids = self.ids[idx]
            if has:
                (fe.move_entities_facing_f32 if f32 else fe.move_entities_facing)(ids, *vals)
            else:
                (fe.move_entities_f32 if f32 else fe.move_entities)(ids, *vals)
            if he is not None:
                (he.move_entities_f32 if f32 else he.move_entities)(ids, vals[0], vals[1])

    def step(self, fe, he, frac=0.5, f32=False, step=35.0):
        """moves and turns a fraction of the entities: a fifth without a facing (it stays), some turn in place, a few ids twice"""
        rng = self.rng
        idx = rng.permutation(self.n)[:max(4, int(self.n * frac))]
        nx = np.clip(self.x[idx] + rng.uniform(-step, step, len(idx)), 0, self.cols * self.w - 1e-3)
        nz = np.clip(self.z[idx] + rng.uniform(-step, step, len(idx)), 0, self.rows * self.w - 1e-3)
        yaw = rng.uniform(0, 2 * np.pi, len(idx))
        nfx, nfz = np.cos(yaw), np.sin(yaw)
        nfx[::11] = nfz[::11] = 0.0  # the facing is dropped
        nfx[5::23] = np.nan          # non-finite: no facing either
        still = np.arange(len(idx)) % 7 == 3  # turn in place
        nx[still], nz[still] = self.x[idx[still]], self.z[idx[still]]
        p = np.arange(len(idx)) % 5 == 0
        f = ~p
        fi = np.concatenate([idx[f], idx[f][:3]])  # three ids twice: the second move wins
        fx2 = np.concatenate([nfx[f], -nfz[f][:3]])
        fz2 = np.concatenate([nfz[f], nfx[f][:3]])
        fxx = np.concatenate([nx[f], nx[f][:3] + 1.0])
        fzz = np.concatenate([nz[f], nz[f][:3]])
        self.events(fe, he, plain=(idx[p], nx[p], nz[p]), facing=(fi, fxx, fzz, fx2, fz2), f32=f32)


def check_follow(chd, W, fe, sel, he_status):
    """chd_get_follow keeps its plain semantics; chd_get_follow_frame equals the restatement bit for bit"""
    capi = chd.capi
    f = fe.get_follow()
    slots = np.array(sorted(W.bind), np.uint32)
    np.testing.assert_array_equal(f["slot"], slots)
    ent = np.array([W.bind[int(s)][0] for s in slots], np.int64)
    np.testing.assert_array_equal(f["entity"], W.ids[ent])
    np.testing.assert_array_equal(bits(f["cx"]), bits(W.x[ent]))
    np.testing.assert_array_equal(bits(f["cz"]), bits(W.z[ent]))
    pos = {s: k for k, s in enumerate(sel)}
    want = np.array([he_status[pos[int(s)]] if int(s) in pos else capi.FOLLOW_NOT_SELECTED if W.live[W.bind[int(s)][0]] else capi.FOLLOW_NO_ENTITY
                     for s in slots], np.uint32)
    np.testing.assert_array_equal(f["status"], want)
    assert f["n_selected"] == len(sel)
    g = fe.get_follow_frame()
    fs = sorted(W.frame)
    np.testing.assert_array_equal(g["slot"], np.array(fs, np.uint32))
    for j, a in enumerate(("fx", "fz", "cx", "cz", "dx", "dz")):
        np.testing.assert_array_equal(bits(g[a]), bits(np.array([W.gen[s][j] for s in fs])), err_msg=a)


def framed_world(chd, W, fe, S, every=2):
    """followers of mixed kinds on every `every`-th slot; two thirds of them framed: zero and non-zero offsets, identity and
    non-identity rotations"""
    slots = np.arange(0, S, every, dtype=np.uint32)
    ent = W.rng.permutation(W.n)[:len(slots)]
    kind, shape = W.shapes(len(slots))
    W.follow(fe, slots, ent, kind, shape)
    a, b = slots[0::3], slots[1::3]
    W.set_frame(fe, a, W.rng.uniform(-120, 120, len(a)), np.where(np.arange(len(a)) % 2, W.rng.uniform(-60, 60, len(a)), 0.0))
    ang = W.rng.uniform(-np.pi, np.pi, len(b))
    W.set_frame(fe, b, np.where(np.arange(len(b)) % 2, 0.0, 80.0), 0.0, rot=(np.cos(ang), np.sin(ang)))
    return slots


# ------------------------------------------------------------------------------------------------- 1. against the host-packed batch
@pytest.mark.parametrize("mode", [0, 1], ids=["all", "moved"])
@pytest.mark.parametrize("graphs", [True, False], ids=["graphs", "direct"])
def test_framed_followers_equal_host_packed_batch(chd, mode, graphs):
    """12 ticks of moving and turning entities with fan-out: framed followers of mixed kinds beside plain ones; moves with facings in
    f64 and f32.  Every host-facing result and status equals the engine fed the host-packed batch, chd_get_follow_frame equals the
    numpy restatement bit for bit and chd_get_follow keeps its plain semantics."""
    capi = chd.capi
    W = FWorld(chd, 4000)
    S = 600
    fe, he = W.engine(S, True, max_pairs=1 << 17), W.engine(S, False, max_pairs=1 << 17)
    for e in (fe, he):
        e.enable_graphs(graphs)
    framed_world(chd, W, fe, S)
    state = None
    for t in range(1, 13):
        if t > 1:
            W.step(fe, he, frac=0.3, f32=bool(t % 2))
        state, off, arr, snd, idx, cmi = rings(chd, W, t, S, state)
        for e in (fe, he):
            e.set_rings(off, arr, snd, idx, cmi)
        fe.follow_queries(mode)
        if t % 2:
            sf = fe.tick(None, t * TICK, capi.TICK_ALL | capi.TICK_FOLLOW)
        else:
            fe.begin_interest(None, t * TICK)
            sf = fe.tick(None, t * TICK, capi.TICK_ALL)
        sel = W.select(mode)
        batch, keep = W.pack(sel)
        sh = he.tick(batch, t * TICK, capi.TICK_ALL)
        assert_same(snapshot(fe, sf), snapshot(he, sh), "tick %d" % t)
        hs = he.get_query_status(len(sel))
        np.testing.assert_array_equal(fe.get_query_status(len(sel)), hs)
        check_follow(chd, W, fe, sel, hs)
        if mode == capi.FOLLOW_MOVED and t > 1:
            assert 0 < len(sel) < len(W.bind)
    assert sf.n_due > 0 and sf.n_kept > 0
    fe.close(), he.close()


# ------------------------------------------------------------------------------------------------- 2. MOVED selection
def test_moved_selects_exactly_the_followers_that_moved_or_turned(chd):
    capi = chd.capi
    W = FWorld(chd, 300, seed=8)
    S = 12
    fe, he = W.engine(S, True), W.engine(S, False)
    slots = np.arange(S, dtype=np.uint32)
    ent = np.arange(S) * 5
    W.fx[ent], W.fz[ent] = 1.0, 0.0
    W.events(fe, he, facing=(ent, W.x[ent], W.z[ent], W.fx[ent], W.fz[ent]))
    kind, shape = W.shapes(S)
    W.follow(fe, slots, ent, kind, shape)
    W.set_frame(fe, slots[:10], 60.0, 20.0)  # slots 10, 11 are plain

    def tick(t):
        fe.follow_queries(capi.FOLLOW_MOVED)
        sf = fe.tick(None, t * TICK, capi.TICK_ALL | capi.TICK_FOLLOW)
        sel = W.select(capi.FOLLOW_MOVED)
        batch, keep = W.pack(sel)
        sh = he.tick(batch, t * TICK, capi.TICK_ALL)
        assert_same(snapshot(fe, sf), snapshot(he, sh), "tick %d" % t)
        hs = he.get_query_status(len(sel))
        check_follow(chd, W, fe, sel, hs)
        return sel

    assert tick(1) == list(range(S))
    assert tick(2) == []
    e = lambda s: int(ent[s])  # noqa: E731
    # 0: turns in place; 10: a plain follower's entity turns in place (not selected); 1: a plain move to the same place keeps the
    # facing (not selected); 2: a plain move elsewhere keeps the facing (selected, the old facing); 3: two facing moves to the same
    # place, the last back to the old facing (not selected); 4: two, the last a new facing (selected)
    k = [e(0), e(10), e(3), e(3), e(4), e(4)]
    W.events(fe, he, plain=(np.array([e(1)]), W.x[[e(1)]], W.z[[e(1)]]))
    W.events(fe, he, plain=(np.array([e(2)]), W.x[[e(2)]] + 7.0, W.z[[e(2)]]))
    W.events(fe, he, facing=(np.array(k), W.x[k], W.z[k], np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.6]), np.array([1.0, 1.0, 1.0, 0.0, 1.0, 0.8])))
    assert tick(3) == [0, 2, 4]
    assert (W.gen[2][0], W.gen[2][1]) == (1.0, 0.0) and (W.gen[4][0], W.gen[4][1]) == (0.6, 0.8)
    # f32: the facings widen exactly
    W.events(fe, he, facing=(np.array([e(5)]), W.x[[e(5)]], W.z[[e(5)]], np.array([0.1]), np.array([0.9])), f32=True)
    assert tick(4) == [5] and W.gen[5][0] == float(np.float32(0.1))
    fe.close(), he.close()


# ------------------------------------------------------------------------------------------------- 3. facing lifecycle
def test_facing_and_frame_lifecycle(chd):
    capi = chd.capi
    W = FWorld(chd, 200, seed=4)
    S = 16
    fe, he = W.engine(S, True, max_subscribers=20), W.engine(S, False, max_subscribers=20)
    slots = np.arange(8, dtype=np.uint32)
    ent = np.arange(8) * 2 + 1
    kind, shape = W.shapes(8)
    W.follow(fe, slots, ent, kind, shape)
    W.set_frame(fe, slots, 90.0, -30.0, rot=(np.zeros(8), np.ones(8)))

    def tick(t, mode=capi.FOLLOW_ALL):
        fe.follow_queries(mode)
        sf = fe.tick(None, t * TICK, capi.TICK_ALL | capi.TICK_FOLLOW)
        sel = W.select(mode)
        batch, keep = W.pack(sel)
        sh = he.tick(batch, t * TICK, capi.TICK_ALL)
        assert_same(snapshot(fe, sf), snapshot(he, sh), "tick %d" % t)
        check_follow(chd, W, fe, sel, he.get_query_status(len(sel)))

    tick(1)
    # a spawn without a facing generates plain; a despawned id's table slot, reused by a spawn without a facing, does not inherit one
    k = int(ent[0])
    assert W.fx[k] != 0.0 or W.fz[k] != 0.0
    for e in (fe, he):
        assert (e.despawn_entities(W.ids[[k]]) == 0).all()
        assert (e.spawn_entities(np.array([900_001], np.uint32), np.array([400.0]), np.array([500.0])) == 0).all()  # (takes k's slot)
    W.ids = np.concatenate([W.ids, [900_001]]).astype(np.uint32)
    W.x, W.z = np.append(W.x, 400.0), np.append(W.z, 500.0)
    W.fx, W.fz = np.append(W.fx, 0.0), np.append(W.fz, 0.0)
    W.live = np.append(W.live, True)
    W.n += 1
    W.live[k] = False
    W.follow(fe, [8], [W.n - 1], [CONE], shape[:, :1])
    W.set_frame(fe, [8], 50.0, 10.0)
    tick(2)
    assert W.gen[8][:2] == (0.0, 0.0) and W.gen[8][2:4] == (400.0, 500.0)
    f = fe.get_follow()
    assert f["status"][0] == capi.FOLLOW_NO_ENTITY
    # re-bind, unbind and remove clear the frame
    W.follow(fe, [1], [ent[1]], kind[1:2], shape[:, 1:2])
    fe.follow_unbind(np.array([2], np.uint32))
    del W.bind[2]
    W.unframe([2])
    for e in (fe, he):
        e.remove_subscribers(np.array([3], np.uint32))
    del W.bind[3]
    W.unframe([3])
    W.bind.pop(0)
    W.unframe([0])
    fe.follow_unbind(np.array([0], np.uint32))
    tick(3)
    assert 1 not in fe.get_follow_frame()["slot"].tolist()
    # a frame on a slot that follows nothing: INVALID, nothing applied
    before = fe.get_follow_frame()
    b = chd.capi.FollowFrameBatch()
    sl = np.array([4, 12], np.uint32)
    v = np.array([5.0, 5.0])
    b.n, b.slot, b.off_fwd = 2, chd.capi.ptr(sl), chd.capi.ptr(v)
    assert fe.L.chd_follow_set_frame(fe.h, C.byref(b)) == capi.ERR_INVALID
    assert "follows nothing" in fe.L.chd_last_error(fe.h).decode()
    # ... and a non-finite offset or rotation on a bound slot
    for field in ("off_fwd", "off_right", "rot_cos"):
        b = chd.capi.FollowFrameBatch()
        sl, v, one = np.array([4], np.uint32), np.array([np.nan]), np.array([1.0])
        b.n, b.slot, b.rot_cos, b.rot_sin = 1, chd.capi.ptr(sl), chd.capi.ptr(one), chd.capi.ptr(one)
        setattr(b, field, chd.capi.ptr(v))
        assert fe.L.chd_follow_set_frame(fe.h, C.byref(b)) == capi.ERR_INVALID, field
        assert "non-finite" in fe.L.chd_last_error(fe.h).decode()
    after = fe.get_follow_frame()
    for a in before:
        np.testing.assert_array_equal(before[a], after[a])
    tick(4, capi.FOLLOW_MOVED)
    # chd_set_subscribers clears every binding and frame
    fe.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
    assert len(fe.get_follow_frame()["slot"]) == 0 and len(fe.get_follow()["slot"]) == 0
    fe.close(), he.close()


# ------------------------------------------------------------------------------------------------- 4. merged batches, pipelined loop
def test_merged_batch_with_framed_followers(chd):
    """chd_follow_queries_with: a host part for the slots that follow nothing (one of them overriding a framed follower) in front of
    the framed followers' generated entries equals one host-packed batch of both."""
    capi = chd.capi
    W = FWorld(chd, 3000, seed=12)
    S = 500
    fe, he = W.engine(S, True, max_pairs=1 << 17, max_queries=1024), W.engine(S, False, max_pairs=1 << 17, max_queries=1024)
    framed_world(chd, W, fe, S)
    for t in range(1, 7):
        if t > 1:
            W.step(fe, he, frac=0.3, f32=bool(t % 2))
        r = np.random.default_rng(50 + t)
        hsub = np.concatenate([np.arange(1, S, 2)[:40 + 5 * t], [0]]).astype(np.uint32)  # slot 0 is a framed follower: overridden
        hx, hz, hr = r.uniform(0, 1600, len(hsub)), r.uniform(0, 1600, len(hsub)), r.uniform(30, 150, len(hsub))
        hb, hk = chd.engine.make_batch(len(hsub), sub=hsub, sphere=(hx, hz, hr))
        fe.follow_queries_with(capi.FOLLOW_MOVED, hb)
        sf = fe.tick(None, t * TICK, capi.TICK_ALL | capi.TICK_FOLLOW)
        W.dirty.add(0)  # (the overridden follower is selected again by the next generation)
        sel = [s for s in W.select(capi.FOLLOW_MOVED) if s != 0]
        q = W.queries(sel)[0].T
        sh_ = np.array([W.bind[s][2] for s in sel]).reshape(len(sel), 7).T
        kind = np.concatenate([np.full(len(hsub), SPHERE, np.uint8), [W.bind[s][1] for s in sel]]).astype(np.uint8)
        cx, cz = np.concatenate([hx, q[:, 2]]), np.concatenate([hz, q[:, 3]])
        z0 = np.zeros(len(hsub))
        batch, keep = chd.engine.make_batch(len(hsub) + len(sel), sub=np.concatenate([hsub, sel]).astype(np.uint32), kind=kind,
                                            sphere=(cx, cz, np.concatenate([hr, sh_[0]])), box=(cx, cz, np.concatenate([z0, sh_[1]]), np.concatenate([z0, sh_[2]])),
                                            cone=(cx, cz, np.concatenate([z0, q[:, 4]]), np.concatenate([z0, q[:, 5]]), np.concatenate([z0, sh_[5]]),
                                                  np.concatenate([z0, sh_[6]])))
        sh = he.tick(batch, t * TICK, capi.TICK_ALL)
        assert_same(snapshot(fe, sf), snapshot(he, sh), "tick %d" % t)
        f = fe.get_follow()
        assert f["status"][0] == capi.FOLLOW_OVERRIDDEN
        g = fe.get_follow_frame()
        fs = [s for s in sorted(W.frame) if s != 0]
        got = {int(s): k for k, s in enumerate(g["slot"])}
        for j, a in enumerate(("fx", "fz", "cx", "cz", "dx", "dz")):
            np.testing.assert_array_equal(bits(g[a][[got[s] for s in fs]]), bits(np.array([W.gen[s][j] for s in fs])), err_msg=a)
    fe.close(), he.close()


def test_pipelined_loop_with_facings_equals_serial(chd):
    """move_entities_facing_f32 -> follow_queries(MOVED) -> begin_interest(NULL) -> tick -> fetch_results_async with the next tick
    enqueued before the wait gives the serial form's results, list by list."""
    capi, torch = chd.capi, chd.torch
    W = FWorld(chd, 20_000, seed=21)
    W.x, W.z = W.x.astype(np.float32).astype(np.float64), W.z.astype(np.float32).astype(np.float64)
    W.fx, W.fz = W.fx.astype(np.float32).astype(np.float64), W.fz.astype(np.float32).astype(np.float64)
    S = 3000
    lim = dict(max_pairs=1 << 18, max_visible=1 << 24)
    pe, se = W.engine(S, True, **lim), W.engine(S, True, **lim)
    framed_world(chd, W, None, S, every=1)
    for e in (pe, se):
        W.apply(e)
    L = pe.L
    P = 1 << 18

    def result_set():
        keep = dict(off=torch.zeros(S + 1, dtype=torch.int32).pin_memory(), ch=torch.zeros(P, dtype=torch.int32).pin_memory(),
                    dist=torch.zeros(P, dtype=torch.int32).pin_memory(), status=torch.zeros(S, dtype=torch.int32).pin_memory(),
                    hdr=torch.zeros(64, dtype=torch.int32).pin_memory())
        r = capi.ResultBuffers()
        r.pair_off, r.pair_channel, r.pair_dist, r.pair_cap = capi.ptr(keep["off"]), capi.ptr(keep["ch"]), capi.ptr(keep["dist"]), P
        r.query_status, r.status_cap = capi.ptr(keep["status"]), S
        return r, keep

    sets = [result_set(), result_set()]
    moves = []
    for t in range(8):
        sel = W.rng.permutation(W.n)[:W.n // 10]
        yaw = W.rng.uniform(0, 2 * np.pi, len(sel))
        moves.append((W.ids[sel].copy(), (W.x[sel] + W.rng.uniform(-30, 30, len(sel))).clip(0, 1599).astype(np.float32),
                      (W.z[sel] + W.rng.uniform(-30, 30, len(sel))).clip(0, 1599).astype(np.float32), np.cos(yaw).astype(np.float32),
                      np.sin(yaw).astype(np.float32)))
    serial = []
    for t, mv in enumerate(moves, 1):
        se.move_entities_facing_f32(*mv)
        se.follow_queries(capi.FOLLOW_MOVED)
        se.begin_interest(None, t * TICK, False)
        s = se.tick(None, t * TICK, capi.TICK_BUILD | capi.TICK_EMIT)
        p = se.get_pairs()
        serial.append(dict(summary=s.as_dict(), off=p["off"], ch=p["channel"], dist=p["dist"], status=se.get_query_status(S)))

    def check(t, summ):
        want, (r, k) = serial[t], sets[t % 2]
        assert {f: getattr(summ, f) for f in want["summary"]} == want["summary"], t
        n = summ.n_pairs
        np.testing.assert_array_equal(k["off"].numpy().view(np.uint32), want["off"])
        np.testing.assert_array_equal(k["ch"].numpy().view(np.uint32)[:n], want["ch"])
        np.testing.assert_array_equal(k["dist"].numpy().view(np.uint32)[:n], want["dist"])
        np.testing.assert_array_equal(k["status"].numpy().view(np.uint32), want["status"])

    summ = capi.TickSummary()
    for t, mv in enumerate(moves):
        pe.move_entities_facing_f32(*mv)
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
    ga, gb = pe.get_follow_frame(), se.get_follow_frame()
    for a in ga:
        np.testing.assert_array_equal(ga[a], gb[a])
    pe.close(), se.close()


def test_pipelined_adopted_merge_with_facings_equals_serial(chd):
    """Explicit rows prefetched a tick ahead (both staging sets in use), adopted and merged with the framed followers
    (chd_follow_queries_with(NULL)), ticked and read back with chd_fetch_results_async while the next tick is enqueued, with the moves
    carrying facings: list by list the results of the serial form with the rows given directly, and the same frame read-back."""
    from tests.test_gpu_follow_merged import result_set

    capi, torch, engine = chd.capi, chd.torch, chd.engine
    W = FWorld(chd, 20_000, seed=23)
    W.x, W.z = W.x.astype(np.float32).astype(np.float64), W.z.astype(np.float32).astype(np.float64)
    W.fx, W.fz = W.fx.astype(np.float32).astype(np.float64), W.fz.astype(np.float32).astype(np.float64)
    S, P = 3000, 1 << 18
    Q = S + 1024
    lim = dict(max_pairs=P, max_visible=1 << 24, max_queries=Q)
    pe, se = W.engine(S, True, **lim), W.engine(S, True, **lim)
    framed_world(chd, W, None, S)
    for e in (pe, se):
        W.apply(e)
    T = 8
    moves = []
    for t in range(T):
        sel = W.rng.permutation(W.n)[:W.n // 10]
        yaw = W.rng.uniform(0, 2 * np.pi, len(sel))
        moves.append((W.ids[sel].copy(), (W.x[sel] + W.rng.uniform(-30, 30, len(sel))).clip(0, 1599).astype(np.float32),
                      (W.z[sel] + W.rng.uniform(-30, 30, len(sel))).clip(0, 1599).astype(np.float32), np.cos(yaw).astype(np.float32),
                      np.sin(yaw).astype(np.float32)))

    def host(t):
        """tick t's explicit rows: slots that follow nothing, and on every third tick a framed follower's override"""
        r = np.random.default_rng(500 + t)
        n_h = [120, 300, 90, 0, 260, 200, 40, 500][t]
        sub = np.arange(1, S, 2)[:n_h]
        if t % 3 == 0:
            sub = np.concatenate([sub, [0]])
        sub = sub.astype(np.uint32)
        return engine.make_batch(len(sub), sub=sub, sphere=(r.uniform(0, 1600, len(sub)), r.uniform(0, 1600, len(sub)), r.uniform(30, 150, len(sub))))

    serial = []
    for t, mv in enumerate(moves):
        se.move_entities_facing_f32(*mv)
        hb, keep = host(t)
        se.follow_queries_with(capi.FOLLOW_MOVED, hb)
        s = se.tick(None, (t + 1) * TICK, capi.TICK_BUILD | capi.TICK_EMIT | capi.TICK_FOLLOW)
        p = se.get_pairs()
        (ns, nc), (us, uc) = se.get_diff(s.n_sub_new, s.n_unsub)
        n = engine.host_part_size(hb.n) + len(W.bind)
        serial.append(dict(summary=s.as_dict(), off=p["off"], ch=p["channel"], dist=p["dist"], new=sorted(zip(ns.tolist(), nc.tolist())),
                           unsub=sorted(zip(us.tolist(), uc.tolist())), status=se.get_query_status(n), voff=se.get_visible()[0],
                           frame=se.get_follow_frame()))
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
    hb, keeps[0] = host(0)
    pe.prefetch_queries(hb, keeps[0])
    for t, mv in enumerate(moves):
        pe.move_entities_facing_f32(*mv)
        pe.adopt_prefetched()
        pe.follow_queries_with(capi.FOLLOW_MOVED, None)  # consumes the adopted rows: their staging set is free again
        if t + 1 < T:  # tick t + 1's rows go into the other staging set while tick t runs
            hb, keeps[(t + 1) % 2] = host(t + 1)
            pe.prefetch_queries(hb, keeps[(t + 1) % 2])
        pe.tick(None, (t + 1) * TICK, capi.TICK_BUILD | capi.TICK_EMIT | capi.TICK_FOLLOW, want_summary=False)
        r, k = sets[t % 2]
        assert pe.L.chd_fetch_results_async(pe.h, C.byref(r), capi.ptr(k["hdr"])) == 0
        if t:
            assert pe.L.chd_fetch_wait(pe.h, C.byref(summ)) == 0
            check(t - 1, summ)
    assert pe.L.chd_fetch_wait(pe.h, C.byref(summ)) == 0
    check(T - 1, summ)
    g, want = pe.get_follow_frame(), serial[-1]["frame"]
    for a in g:
        np.testing.assert_array_equal(bits(g[a]) if a != "slot" else g[a], bits(want[a]) if a != "slot" else want[a])
    pe.close(), se.close()


# ------------------------------------------------------------------------------------------------- 5. scale
@pytest.mark.parametrize("graphs", [True, False], ids=["graphs", "direct"])
def test_scale_one_million_entities_100k_framed_followers(chd, graphs):
    """1 M entities, 100 K framed followers on 600 K slots: the generation spans more tiles than the device has SMs."""
    capi = chd.capi
    S = 600_000
    sms = chd.torch.cuda.get_device_properties(0).multi_processor_count
    assert (S + 4095) // 4096 > sms
    W = FWorld(chd, 1_000_000, cols=64, rows=64, w=500.0, seed=9)
    lim = dict(max_pairs=4_000_000, max_visible=1 << 20, max_due=1 << 20, max_window_cells=8_000_000)
    fe, he = W.engine(S, True, **lim), W.engine(S, False, **lim)
    for e in (fe, he):
        e.enable_graphs(graphs)
    slots = np.arange(3, S, 6, dtype=np.uint32)[:100_000]
    ent = W.rng.permutation(W.n)[:len(slots)]
    kind, shape = W.shapes(len(slots))
    W.follow(fe, slots, ent, kind, shape)
    ang = W.rng.uniform(-np.pi, np.pi, len(slots))
    W.set_frame(fe, slots, W.rng.uniform(-300, 300, len(slots)), W.rng.uniform(-200, 200, len(slots)), rot=(np.cos(ang), np.sin(ang)))
    for t, mode in ((1, capi.FOLLOW_ALL), (2, capi.FOLLOW_MOVED), (3, capi.FOLLOW_MOVED), (4, capi.FOLLOW_ALL)):
        if t > 1:
            W.step(fe, he, frac=0.05, f32=t == 3, step=200.0)
        fe.follow_queries(mode)
        sf = fe.tick(None, t * TICK, capi.TICK_BUILD | capi.TICK_FOLLOW)
        sel = W.select(mode)
        batch, keep = W.pack(sel)
        sh = he.tick(batch, t * TICK, capi.TICK_BUILD)
        assert_same(snapshot(fe, sf, vis=False), snapshot(he, sh, vis=False), "tick %d" % t)
        check_follow(chd, W, fe, sel, he.get_query_status(len(sel)))
    fe.close(), he.close()


# ------------------------------------------------------------------------------------------------- 6. slabs
class FSlabs(Slabs):
    """Slabs whose entity events carry facings, whose hand-offs carry them through chd_handoff_entities_facing, and whose arriving
    followers get their frames again after the bind."""

    def spawn(self, ids, x, z, fx=None, fz=None):
        for e, b in zip(self.engines, self.router.spawn(ids, x, z, fx, fz)):
            if len(b[0]):
                assert (e.spawn_entities_facing(*b) == 0).all()

    def move(self, ids, x, z, fx=None, fz=None):
        for e, b in zip(self.engines, self.router.move(ids, x, z, fx, fz)):
            if len(b[0]):
                e.move_entities_facing(*b)

    def place(self):
        """Slabs.place, and the frames of the arriving followers set after their bind"""
        for r, v in enumerate(self.vacated):
            self.reg.slots.release(r, v)
        arrivals, out_lists, in_calls, vacated, binds = self.reg.plan(self.router)
        for r, v in enumerate(vacated):
            if v:
                self.engines[r].remove_subscribers(v)
        moved = set()
        for dst, src, first, pairs in in_calls:
            self.engines[dst].add_subscribers([s for _, s in pairs], [c for c, _ in pairs])
            moved |= {c for c, _ in pairs}
        for r, a in enumerate(arrivals):
            if a:
                self.engines[r].add_subscribers([s for _, s in a], [c for c, _ in a])
        for r, b in enumerate(binds):
            if len(b["conn"]):
                _bind(self.engines[r], b["slot"], b["entity"], b["kind"], b["shape"])
                if "frame" in b:
                    f = b["frame"]
                    self.engines[r].follow_set_frame(f["slot"], f["off_fwd"], f["off_right"], (f["rot_cos"], f["rot_sin"]))
        self.vacated = vacated
        return moved

    def handoff(self):
        lists = []
        for r, e in enumerate(self.engines):
            ids, dst, x, z, fx, fz = e.handoff_entities_facing()  # (no communicator: dst names rank 0; the owner comes from x)
            owner = self.chd.sharding.owner_of_column(self.chd.sharding.column_of(x, 0.0, W, COLS), COLS, self.world)
            assert not (owner == r).any()
            lists.append((ids, owner, x, z, fx, fz))
        for r, b in enumerate(self.router.handoff(lists)):
            if len(b[0]):
                assert (self.engines[r].spawn_entities_facing(*b) == 0).all()
        return [int(i) for l in lists for i in l[0].tolist()]


def _fslab_setup(chd, world, halo_extra, seed, n=6000, F=480, max_off=60.0, halo=None):
    rng = np.random.default_rng(seed)
    walk = Walk(n, seed)
    yaw = rng.uniform(0, 2 * np.pi, n)
    fx, fz = np.cos(yaw), np.sin(yaw)
    fol_ids = rng.choice(walk.ids, F, replace=False)
    kind, shape = _shapes(rng, F)
    frames = np.stack([rng.uniform(-max_off, max_off, F), rng.uniform(-max_off, max_off, F), np.ones(F), np.zeros(F)])
    ang = rng.uniform(-np.pi, np.pi, F)
    frames[2, 1::2], frames[3, 1::2] = np.cos(ang[1::2]), np.sin(ang[1::2])
    if halo is None:  # the reach and the offset
        halo = chd.sharding.halo_columns(180.0 + max_off * np.sqrt(2), W) + halo_extra
    sl = FSlabs(chd, world, halo, n, F)
    whole = chd.engine.Engine(_cfg(chd), 2 * n, F, max_visible=1 << 24)
    whole.entity_table_init()
    whole.set_subscribers(np.arange(1, F + 1, dtype=np.uint32))
    assert (whole.spawn_entities_facing(walk.ids, walk.x, walk.z, fx, fz) == 0).all()
    sl.spawn(walk.ids, walk.x, walk.z, fx, fz)
    _bind(whole, np.arange(F), fol_ids, kind, shape)
    whole.follow_set_frame(np.arange(F, dtype=np.uint32), frames[0], frames[1], (frames[2], frames[3]))
    for j in range(F):
        sl.reg.follow(j + 1, int(fol_ids[j]), int(kind[j]), shape[:, j], frame=tuple(frames[:, j]))
    return walk, fx, fz, fol_ids, kind, shape, frames, halo, sl, whole


def _turn(walk, fx, fz, rng):
    ids, x, z = walk.tick()
    yaw = rng.uniform(0, 2 * np.pi, len(ids))
    fx[ids - 1], fz[ids - 1] = np.cos(yaw), np.sin(yaw)
    return ids, x, z, fx[ids - 1].copy(), fz[ids - 1].copy()


@pytest.mark.parametrize("world", [2, 3])
def test_framed_followers_on_slabs_equal_the_whole_world(chd, world):
    """Framed followers; entities walk and turn across slab borders and are handed off with their facings.  Every tick, per
    connection, the visible set, the pairs and the follower's status equal a whole-world engine's."""
    capi = chd.capi
    walk, fx, fz, fol_ids, kind, shape, frames, halo, sl, whole = _fslab_setup(chd, world, 1, 140 + world)
    rng = np.random.default_rng(7)
    F = len(fol_ids)
    handed = 0
    for t in range(8):
        if t:
            mv = _turn(walk, fx, fz, rng)
            whole.move_entities_facing(*mv)
            sl.move(*mv)
        moved = sl.place()
        whole.follow_queries(capi.FOLLOW_MOVED)
        assert whole.tick(None, (t + 1) * TICK, 1 | 2 | capi.TICK_FOLLOW).overflow == 0
        sl.tick((t + 1) * TICK, capi.FOLLOW_MOVED)
        wr = _results(whole)
        per = [_results(e) for e in sl.engines]
        wf = whole.get_follow_frame()
        for c in range(1, F + 1):
            r = sl.reg.owner_of(c)
            got, want = per[r][sl.reg.slots.slot[c]], wr[c - 1]
            why = (t, c, r, c in moved, got["follow"], want["follow"])
            if want["follow"][1] != capi.Q_OK:  # an offset centre out of the world fails the query: both keep the pairs they had, which
                assert got["follow"][1] == want["follow"][1], why  # differ once the connection moved rank or was outside its slab
                continue
            assert got["vis"] == want["vis"], why
            assert got["pairs"] == want["pairs"], why
            assert got["follow"][1] != capi.FOLLOW_OUTSIDE_SLAB, why
            if c not in moved:
                assert got["follow"] == want["follow"], (t, c)
        for r, e in enumerate(sl.engines):  # the framed queries of each rank equal the whole world's for its connections
            g = e.get_follow_frame()
            for k, s in enumerate(g["slot"].tolist()):
                c = sl.reg.slots.at[r][s]
                if c in moved:
                    continue
                for a in ("fx", "fz", "cx", "cz", "dx", "dz"):
                    assert bits(g[a][k]) == bits(wf[a][c - 1]), (t, c, a)
        handed += len(set(sl.handoff()) & set(fol_ids.tolist()))
    assert handed > 0
    sl.close(), whole.close()


def test_minimal_halo_outside_slab_follows_the_offset_centre(chd):
    """halo = halo_columns(reach + offset): OUTSIDE_SLAB appears exactly where a numpy span of the offset centre says."""
    capi, world = chd.capi, 3
    walk, fx, fz, fol_ids, kind, shape, frames, halo, sl2, whole = _fslab_setup(chd, world, 0, 177, max_off=150.0, halo=chd.sharding.halo_columns(180.0, W))
    slabs = [chd.sharding.slab_columns(COLS, world, r) for r in range(world)]
    rng = np.random.default_rng(8)
    seen = 0
    for t in range(6):
        if t:
            mv = _turn(walk, fx, fz, rng)
            whole.move_entities_facing(*mv)
            sl2.move(*mv)
        moved = sl2.place()
        whole.follow_queries(capi.FOLLOW_ALL)
        whole.tick(None, (t + 1) * TICK, 1 | 2 | capi.TICK_FOLLOW)
        sl2.tick((t + 1) * TICK, capi.FOLLOW_ALL)
        wr = _results(whole)
        per = [_results(e) for e in sl2.engines]
        for c in range(1, len(fol_ids) + 1):
            r = sl2.reg.owner_of(c)
            k = fol_ids[c - 1] - 1
            f = frames[:, c - 1]
            cx = float(frame_query(walk.x[k], walk.z[k], fx[k], fz[k], *f, 0.0, 0.0)[2])
            side = _outside(cx, int(kind[c - 1]), shape[:, c - 1], slabs[r][0], slabs[r][1], halo)
            got, want = per[r][sl2.reg.slots.slot[c]], wr[c - 1]
            why = (t, c, r, cx, walk.x[k], got["follow"], want["follow"])
            if side:
                seen += 1
                assert got["follow"][1] == capi.FOLLOW_OUTSIDE_SLAB, why
            else:
                assert got["follow"][1] != capi.FOLLOW_OUTSIDE_SLAB, why
                if want["follow"][1] != capi.Q_OK:  # (a failed query, as in the test above)
                    assert got["follow"][1] == want["follow"][1], why
                    continue
                assert got["pairs"] == want["pairs"], why
        sl2.handoff()
    assert seen > 0
    sl2.close(), whole.close()


@pytest.mark.parametrize("graphs", [True, False], ids=["graphs", "direct"])
def test_tick_sharded_with_framed_followers_at_world_one(chd, graphs):
    capi = chd.capi
    n, S, F = 4000, 300, 200
    walk = Walk(n, 19, step=40.0)
    rng = np.random.default_rng(20)
    yaw = rng.uniform(0, 2 * np.pi, n)
    fx, fz = np.cos(yaw), np.sin(yaw)
    kind, shape = _shapes(rng, F)
    fol = rng.choice(walk.ids, F, replace=False)
    sh = chd.engine.Engine(_cfg(chd), 3 * n + 16, S, max_visible=1 << 24, max_queries=1024)
    one = chd.engine.Engine(_cfg(chd), 3 * n + 16, S, max_visible=1 << 24, max_queries=1024)
    sh.comm_init(chd.engine.Engine.comm_unique_id(), 0, 1, 2, n)
    for e in (sh, one):
        e.enable_graphs(graphs)
        e.entity_table_init()
        e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
        assert (e.spawn_entities_facing(walk.ids, walk.x, walk.z, fx, fz) == 0).all()
        _bind(e, np.arange(F), fol, kind, shape)
        e.follow_set_frame(np.arange(0, F, 2, dtype=np.uint32), 40.0, -25.0, (np.zeros(F // 2), np.ones(F // 2)))
    for t in range(6):
        if t:
            mv = _turn(walk, fx, fz, rng)
            for e in (sh, one):
                e.move_entities_facing(*mv)
        for e in (sh, one):
            e.follow_queries(capi.FOLLOW_MOVED)
        s1 = sh.tick_sharded(None, (t + 1) * TICK, capi.TICK_ALL | capi.TICK_FOLLOW)
        s2 = one.tick(None, (t + 1) * TICK, capi.TICK_ALL | capi.TICK_FOLLOW)
        assert _summary_fields(s1) == _summary_fields(s2), t
        a, b = snapshot(sh, s1, vis=False), snapshot(one, s2, vis=False)
        a["summary"], b["summary"] = None, None
        assert_same(a, b, "tick %d" % t)
        assert _vis_sets(*sh.get_visible()) == _vis_sets(*one.get_visible()), t
        ga, gb = sh.get_follow_frame(), one.get_follow_frame()
        for k in ga:
            np.testing.assert_array_equal(ga[k], gb[k])
        assert len(ga["slot"]) == F // 2
    assert chd.capi.lib().chd_comm_destroy(sh.h) == capi.OK
    sh.close(), one.close()


# ------------------------------------------------------------------------------------------------- 7. rules and no change
def test_index_mode_refuses_every_facing_call(chd):
    capi = chd.capi
    e = chd.engine.Engine(chd.engine.grid_cfg(0, 0, 100, 100, 8, 8), 100, 8)
    e.set_subscribers(np.arange(1, 9, dtype=np.uint32))
    e.set_entities(np.full(100, 50.0), np.full(100, 50.0))
    e.follow_bind(np.array([0], np.uint32), np.array([3], np.uint32), sph_r=np.array([40.0]))
    one = np.array([1], np.uint32)
    d = np.array([1.0])
    f = np.array([1.0], np.float32)
    n = C.c_uint32()
    b = capi.FollowFrameBatch(n=1, slot=capi.ptr(np.array([0], np.uint32)))
    for fn, args in (("chd_spawn_entities_facing", (capi.ptr(one), capi.ptr(d), capi.ptr(d), capi.ptr(d), capi.ptr(d), 1, None)),
                     ("chd_spawn_entities_facing_f32", (capi.ptr(one), capi.ptr(f), capi.ptr(f), capi.ptr(f), capi.ptr(f), 1, None)),
                     ("chd_move_entities_facing", (capi.ptr(one), capi.ptr(d), capi.ptr(d), capi.ptr(d), capi.ptr(d), 1)),
                     ("chd_move_entities_facing_f32", (capi.ptr(one), capi.ptr(f), capi.ptr(f), capi.ptr(f), capi.ptr(f), 1)),
                     ("chd_handoff_entities_facing", (None, None, None, None, None, None, 0, C.byref(n))),
                     ("chd_follow_set_frame", (C.byref(b),)),
                     ("chd_get_follow_frame", (None, None, None, None, None, None, None, 0, C.byref(n)))):
        refused(e, capi.ERR_STATE, None, fn, *args)
    assert "entity-table mode" in e.L.chd_last_error(e.h).decode()
    e.close()


@pytest.mark.parametrize("graphs", [True, False], ids=["graphs", "direct"])
def test_plain_followers_run_unchanged_beside_the_frame_paths(chd, graphs):
    """Two table engines run the same plain-follower ticks; one first made (and cleared) a frame on an unrelated slot.  Launch and
    graph-replay counts per tick are equal, and so are the generated batches' results, bit for bit."""
    capi = chd.capi
    W = FWorld(chd, 3000, seed=30)
    S = 400
    a, b = W.engine(S, False), W.engine(S, False)
    for e in (a, b):
        e.enable_graphs(graphs)
    b.follow_bind(np.array([S - 1], np.uint32), W.ids[[5]], sph_r=np.array([50.0]))
    b.follow_set_frame(np.array([S - 1], np.uint32), 30.0, 0.0)
    b.follow_unbind(np.array([S - 1], np.uint32))
    assert len(b.get_follow_frame()["slot"]) == 0
    slots = np.arange(0, S - 1, 2, dtype=np.uint32)
    ent = W.rng.permutation(W.n)[:len(slots)]
    kind, shape = W.shapes(len(slots))
    for e in (a, b):
        e.follow_bind(slots, W.ids[ent], kind=kind, sph_r=shape[0], box=(shape[1], shape[2]), cone=tuple(shape[3:7]))
    for t in range(1, 9):
        if t > 1:
            idx = W.rng.permutation(W.n)[:300]
            nx, nz = W.x[idx] + W.rng.uniform(-30, 30, 300), W.z[idx] + W.rng.uniform(-30, 30, 300)
            for e in (a, b):
                e.move_entities(W.ids[idx], nx, nz)
        counts = []
        for e in (a, b):
            l0, g0 = e.launch_count(), e.graph_launch_count()
            e.follow_queries(capi.FOLLOW_MOVED if t % 2 else capi.FOLLOW_ALL)
            s = e.tick(None, t * TICK, capi.TICK_ALL | capi.TICK_FOLLOW)
            counts.append((e.launch_count() - l0, e.graph_launch_count() - g0, s))
        assert counts[0][:2] == counts[1][:2], (t, counts[0][:2], counts[1][:2])
        assert_same(snapshot(a, counts[0][2]), snapshot(b, counts[1][2]), "tick %d" % t)
        fa, fb = a.get_follow(), b.get_follow()
        for k in ("slot", "entity", "status", "cx", "cz"):
            np.testing.assert_array_equal(fa[k], fb[k])
        np.testing.assert_array_equal(a.get_query_status(len(slots)), b.get_query_status(len(slots)))
    a.close(), b.close()
