"""Visible-set deltas (chd_visible_delta / CHD_TICK_VISIBLE_DELTA): per subscriber slot the entities that entered / left its
visible set since the last successful delta, checked against set differences of the oracle's (or the engine's own) visible lists.
Run on an H100:  python -m pytest tests -m gpu"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

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


def _oracle_grid(wc):
    from tests._oracle import make_grid

    return make_grid(wc.offx, wc.offz, wc.w, wc.h, wc.cols, wc.rows, wc.server_cols, wc.server_rows)


def _pad(off, n):
    """visible offsets of fewer slots -> n + 1 offsets (the extra slots see nothing)"""
    off = np.asarray(off, np.uint64)
    return np.concatenate([off, np.full(n + 1 - len(off), off[-1], np.uint64)]) if len(off) < n + 1 else off


def _set_diff(prev, now, n):
    """(vis_off, vis_entity) before and after -> (enter_off, enter, leave_off, leave) in the order the engine defines"""
    def keys(v):
        off, ent = _pad(v[0], n), np.asarray(v[1], np.uint64)
        slot = np.repeat(np.arange(n, dtype=np.uint64), np.diff(off).astype(np.int64))
        return slot, (slot << np.uint64(32)) | ent

    ps, pk = keys(prev)
    ns, nk = keys(now)
    ent_mask, left_mask = ~np.isin(nk, pk), ~np.isin(pk, nk)
    eo = np.concatenate([[0], np.cumsum(np.bincount(ns[ent_mask].astype(np.int64), minlength=n))]).astype(np.uint64)
    lo = np.concatenate([[0], np.cumsum(np.bincount(ps[left_mask].astype(np.int64), minlength=n))]).astype(np.uint64)
    return eo, (nk[ent_mask] & np.uint64(0xFFFFFFFF)).astype(np.uint32), lo, (pk[left_mask] & np.uint64(0xFFFFFFFF)).astype(np.uint32)


def _assert_delta(got, want):
    eo, en, lo, le = got
    n = len(want[0]) - 1
    np.testing.assert_array_equal(_pad(eo, n), want[0])
    np.testing.assert_array_equal(en, want[1])
    np.testing.assert_array_equal(_pad(lo, n), want[2])
    np.testing.assert_array_equal(le, want[3])


EMPTY = (np.zeros(1, np.uint64), np.zeros(0, np.uint32))


def _world(chd, name, n_ent=None, n_sub=None, radius=None):
    wc = chd.synth.CONFIGS[name] if n_ent is None else chd.synth.scaled(chd.synth.CONFIGS[name], n_ent, n_sub)
    ex, ez = chd.synth.entities(wc)
    S, N = wc.n_subscribers, wc.n_entities
    idx = (np.arange(S, dtype=np.int64) * max(N // S, 1)) % N  # subscriber j stands on entity idx[j]
    r = np.full(S, wc.radius if radius is None else radius)
    return wc, ex, ez, idx, r


def _batch(chd, idx, x, z, r):
    return chd.engine.make_batch(len(idx), sub=np.arange(len(idx), dtype=np.uint32), sphere=(x[idx].copy(), z[idx].copy(), r))


@pytest.mark.parametrize("name,n_ent,n_sub,radius", [("2x2", None, None, 50.0), ("2x2", None, None, 500.0), ("2x2", None, None, 2500.0),
                                                     ("benchmark", 30_000, 3_000, None)])
def test_delta_matches_oracle_set_differences(chd, oracle, name, n_ent, n_sub, radius):
    """12 ticks of moving entities (and the subscribers standing on them): entered / left = set differences of consecutive oracle
    visible lists, as arrays in the engine's order.  The emit kernel is not run: the delta needs only the cell CSR and the pairs."""
    wc, x, z, idx, r = _world(chd, name, n_ent, n_sub, radius)
    og = _oracle_grid(wc)
    S = wc.n_subscribers
    e = chd.engine.Engine(wc.cfg(), wc.n_entities, S)
    e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
    e.reserve_visible_delta(1 << 22)
    prev = EMPTY
    changes = 0
    for t in range(12):
        if t:
            x, z = chd.synth.move_entities(wc, x, z, t, 150.0)
        want = oracle.sphere_tick(og, x, z, x[idx], z[idx], r)
        e.set_entities(x, z)
        batch, keep = _batch(chd, idx, x, z, r)
        e.tick(batch, t * 33 * MS, chd.capi.TICK_BUILD | chd.capi.TICK_VISIBLE_DELTA)
        now = (want["vis_off"], want["vis_entity"])
        d = e.get_visible_delta()
        _assert_delta(d, _set_diff(prev, now, S))
        if t:
            changes += len(d[1]) + len(d[3])
        prev = now
    assert changes > 0


def test_delta_reconstructs_the_visible_lists(chd):
    """Applying left, then entered, to the previous tick's visible lists gives this tick's lists (as sets), for every slot."""
    wc, x, z, idx, r = _world(chd, "benchmark", 30_000, 3_000)
    S = wc.n_subscribers
    e = chd.engine.Engine(wc.cfg(), wc.n_entities, S)
    e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
    e.reserve_visible_delta(1 << 20)
    prev = [set() for _ in range(S)]
    for t in range(8):
        x, z = chd.synth.move_entities(wc, x, z, t, 60.0)
        e.set_entities(x, z)
        batch, keep = _batch(chd, idx, x, z, r)
        e.tick(batch, t * 33 * MS, chd.capi.TICK_BUILD | chd.capi.TICK_EMIT | chd.capi.TICK_VISIBLE_DELTA)
        voff, vis = e.get_visible()
        eo, en, lo, le = e.get_visible_delta()
        for s in range(S):
            left, entered = le[lo[s]:lo[s + 1]], en[eo[s]:eo[s + 1]]
            assert set(left.tolist()) <= prev[s] and not (set(entered.tolist()) & (prev[s] - set(left.tolist())))
            cur = (prev[s] - set(left.tolist())) | set(entered.tolist())
            assert cur == set(vis[voff[s]:voff[s + 1]].tolist()), (t, s)
            prev[s] = cur


def test_delta_spans_everything_since_the_last_delta(chd, oracle):
    """Ticks without the flag and standalone chd_build / chd_update_interest between two deltas fold into the next one; a tick
    without a query batch reports only what entity movement changed."""
    wc, x, z, idx, r = _world(chd, "benchmark", 30_000, 3_000)
    og = _oracle_grid(wc)
    S = wc.n_subscribers
    e = chd.engine.Engine(wc.cfg(), wc.n_entities, S)
    e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
    e.reserve_visible_delta(1 << 20)
    e.set_entities(x, z)
    batch, keep = _batch(chd, idx, x, z, r)
    e.tick(batch, 0, chd.capi.TICK_BUILD | chd.capi.TICK_VISIBLE_DELTA)
    w0 = oracle.sphere_tick(og, x, z, x[idx], z[idx], r)
    for t in (1, 2, 3):  # plain ticks
        x, z = chd.synth.move_entities(wc, x, z, t, 100.0)
        e.set_entities(x, z)
        batch, keep = _batch(chd, idx, x, z, r)
        e.tick(batch, t * 33 * MS, chd.capi.TICK_BUILD | chd.capi.TICK_EMIT)
    x, z = chd.synth.move_entities(wc, x, z, 4, 100.0)  # standalone calls
    e.set_entities(x, z)
    e.build()
    batch, keep = _batch(chd, idx, x, z, r)
    e.update_interest(batch, 4 * 33 * MS)
    e.visible_delta()
    w1 = oracle.sphere_tick(og, x, z, x[idx], z[idx], r)
    _assert_delta(e.get_visible_delta(), _set_diff((w0["vis_off"], w0["vis_entity"]), (w1["vis_off"], w1["vis_entity"]), S))
    # no query batch: the subscriptions stay where they were, only the entities move
    qx, qz = x[idx].copy(), z[idx].copy()
    x, z = chd.synth.move_entities(wc, x, z, 5, 100.0)
    e.set_entities(x, z)
    e.tick(None, 5 * 33 * MS, chd.capi.TICK_BUILD | chd.capi.TICK_VISIBLE_DELTA)
    w2 = oracle.sphere_tick(og, x, z, qx, qz, r)
    d = e.get_visible_delta()
    _assert_delta(d, _set_diff((w1["vis_off"], w1["vis_entity"]), (w2["vis_off"], w2["vis_entity"]), S))
    assert len(d[1]) > 0


def test_delta_subscriber_lifecycle_and_entity_count(chd, oracle):
    """Removed slots leave what they saw, added slots enter what their first query shows, a failed query changes nothing; entity
    spawns at the end of the array, a shrunk array and NaN-parked slots come out as enter / leave.  Handover detection keeps its
    rule: skipped when the entity count changes."""
    wc, x, z, idx, r = _world(chd, "benchmark", 20_000, 1_000)
    og = _oracle_grid(wc)
    S = wc.n_subscribers
    F = chd.capi.TICK_BUILD | chd.capi.TICK_EMIT | chd.capi.TICK_VISIBLE_DELTA
    e = chd.engine.Engine(wc.cfg(), 30_000, S + 8)
    e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
    e.reserve_visible_delta(1 << 20)
    e.set_entities(x, z)
    batch, keep = _batch(chd, idx, x, z, r)
    e.tick(batch, 0, F)
    prev = e.get_visible()

    def step(t, batch, n_slots):
        s = e.tick(batch, t * 33 * MS, F)
        now = e.get_visible()
        d = e.get_visible_delta()
        _assert_delta(d, _set_diff(prev, now, n_slots))
        return s, now, d

    # remove slots 3 and 7: they leave their whole lists and enter nothing
    e.remove_subscribers([3, 7])
    s, now, d = step(1, batch, S)
    for slot in (3, 7):
        np.testing.assert_array_equal(d[3][d[2][slot]:d[2][slot + 1]], prev[1][prev[0][slot]:prev[0][slot + 1]])
        assert d[0][slot] == d[0][slot + 1] and now[0][slot] == now[0][slot + 1]
    prev = now
    # add slots S and S+1 with a first query; slot 0's query fails (radius 0): it keeps its subscriptions, so no change for it
    e.add_subscribers([S, S + 1], [9001, 9002])
    sub = np.array([0, S, S + 1], np.uint32)
    qb, keep = chd.engine.make_batch(3, sub=sub, sphere=(np.array([x[0], x[5], x[9]]), np.array([z[0], z[5], z[9]]), np.array([0.0, 300.0, 300.0])))
    s, now, d = step(2, qb, S + 2)
    assert e.get_query_status(3)[0] == chd.capi.Q_ERR_BAD_STEP
    assert d[0][0] == d[0][1] and d[2][0] == d[2][1]
    for slot in (S, S + 1):
        np.testing.assert_array_equal(d[1][d[0][slot]:d[0][slot + 1]], now[1][now[0][slot]:now[0][slot + 1]])
        assert now[0][slot + 1] > now[0][slot]
    prev = now
    # spawn 5000 entities at the end of the array: no handover detection on a count change
    gx, gz = chd.synth.entities(chd.synth.scaled(wc, 25_000, S))
    x, z = np.concatenate([x, gx[20_000:]]), np.concatenate([z, gz[20_000:]])
    e.set_entities(x, z)
    s, now, d = step(3, None, S + 2)
    assert s.n_handover == 0 and len(d[1]) > 0 and len(d[3]) == 0 and (d[1] >= 20_000).all()
    prev = now
    # same count, some entities parked at NaN and the rest moving: handovers as before, parked ones leave
    x2, z2 = chd.synth.move_entities(wc, x, z, 4, 100.0)
    x2[::97] = np.nan
    e.set_entities(x2, z2)
    s, now, d = step(4, None, S + 2)
    moved = np.nonzero(oracle.cell_of(og, x, z) != oracle.cell_of(og, x2, z2))[0]
    assert s.n_handover == len(moved) > 0
    ho = e.get_handover(s.n_handover)[0]
    np.testing.assert_array_equal(np.sort(ho), moved.astype(np.uint32))
    assert np.isin(np.arange(0, len(x2), 97), d[3]).any()
    prev = now
    # shrink to 12000 entities: everything at or above the new count leaves
    e.set_entities(x2[:12_000], z2[:12_000])
    s, now, d = step(5, None, S + 2)
    assert s.n_handover == 0 and len(d[3]) > 0 and len(d[1]) == 0 and (d[3] >= 12_000).all()


def test_delta_overflow_keeps_the_snapshot(chd):
    """A capacity that is too small raises CHD_OVF_DELTA with the required counts, changes nothing else, and leaves the snapshot
    where it was: after growing the capacity the next delta spans both ticks."""
    wc, x, z, idx, r = _world(chd, "benchmark", 30_000, 3_000)
    S = wc.n_subscribers
    L = chd.capi.lib()
    a = chd.engine.Engine(wc.cfg(), wc.n_entities, S, max_visible=1 << 23)
    b = chd.engine.Engine(wc.cfg(), wc.n_entities, S, max_visible=1 << 23)
    for e in (a, b):
        e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
    ring_state = None
    first = first_v = None
    for t, radius in enumerate((50.0, 1000.0, 1000.0)):  # the larger radius makes the lists of tick 1 outgrow tick 0's
        if t:
            x, z = chd.synth.move_entities(wc, x, z, t, 60.0)
        ring_state, off, arr, snd, ridx, cmi = chd.synth.update_rings(wc, t, t * 33 * MS, 33 * MS, 4, S, ring_len=16, state=ring_state)
        batch, keep = _batch(chd, idx, x, z, np.full(S, radius))
        res = []
        for e, flags in ((b, chd.capi.TICK_ALL), (a, chd.capi.TICK_ALL | chd.capi.TICK_VISIBLE_DELTA)):
            if t == 0 and e is a:
                a.reserve_visible_delta(res[0][1].n_visible)  # exactly the first delta (= the visible lists)
            e.set_entities(x, z)
            e.set_rings(off, arr, snd, ridx, cmi)
            e.tick(batch, t * 33 * MS, flags, want_summary=False)
            s = chd.capi.TickSummary()
            res.append((L.chd_summary(e.h, C.byref(s)), s))
        (stb, sb), (sta, sa) = res
        assert stb == chd.capi.OK
        if t == 1:
            assert sta == chd.capi.ERR_CAPACITY and sa.overflow == chd.capi.OVF_DELTA
            ne, nl, ns = a.visible_delta_counts()
            assert ne > first_v and ns == S
            with pytest.raises(chd.capi.ChdError) as ei:
                a.get_visible_delta()
            assert ei.value.status == chd.capi.ERR_CAPACITY
        else:
            assert sta == chd.capi.OK and sa.overflow == 0
        # everything but the delta is as without it
        assert {k: v for k, v in sa.as_dict().items() if k != "overflow"} == {k: v for k, v in sb.as_dict().items() if k != "overflow"}
        pa, pb = a.get_pairs(), b.get_pairs()
        for k in pa:
            np.testing.assert_array_equal(pa[k], pb[k])
        va, vb = a.get_visible(), b.get_visible()
        np.testing.assert_array_equal(va[0], vb[0])
        np.testing.assert_array_equal(va[1], vb[1])
        assert sorted(a.get_due(sa.n_due).tolist()) == sorted(b.get_due(sb.n_due).tolist())
        for u, v in zip(a.get_handover(sa.n_handover), b.get_handover(sb.n_handover)):
            np.testing.assert_array_equal(np.sort(u), np.sort(v))
        if t == 0:
            first, first_v = va, sa.n_visible
            _assert_delta(a.get_visible_delta(), _set_diff(EMPTY, va, S))
        elif t == 1:
            a.reserve_visible_delta(1 << 23)
        else:
            _assert_delta(a.get_visible_delta(), _set_diff(first, va, S))


def test_delta_leaves_the_tick_unchanged_when_off(chd):
    """Two engines, identical inputs over 6 ticks, one with CHD_TICK_VISIBLE_DELTA: every other result is identical, and an engine
    that reserved the delta but does not ask for it launches exactly what an engine without it launches."""
    wc, x, z, idx, r = _world(chd, "benchmark", 30_000, 3_000)
    S = wc.n_subscribers
    engines = [chd.engine.Engine(wc.cfg(), wc.n_entities, S) for _ in range(3)]
    for e in engines:
        e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
    engines[0].reserve_visible_delta(1 << 20)
    engines[1].reserve_visible_delta(1 << 20)
    flags = [chd.capi.TICK_ALL | chd.capi.TICK_VISIBLE_DELTA, chd.capi.TICK_ALL, chd.capi.TICK_ALL]
    ring_state = None
    for t in range(6):
        x, z = chd.synth.move_entities(wc, x, z, t, 60.0)
        ring_state, off, arr, snd, idx_, cmi = chd.synth.update_rings(wc, t, t * 33 * MS, 33 * MS, 4, S, ring_len=16, state=ring_state)
        batch, keep = _batch(chd, idx, x, z, r)
        res = []
        for e, f in zip(engines, flags):
            e.set_entities(x, z)
            e.set_rings(off, arr, snd, idx_, cmi)
            s = e.tick(batch, t * 33 * MS, f)
            res.append(dict(s=s.as_dict(), pairs=e.get_pairs(), diff=e.get_diff(s.n_sub_new, s.n_unsub), due=e.get_due(s.n_due),
                            vis=e.get_visible(), ho=e.get_handover(s.n_handover), cells=e.get_cells()))
        for other in res[1:]:
            assert other["s"] == res[0]["s"]
            for k in res[0]["pairs"]:
                np.testing.assert_array_equal(other["pairs"][k], res[0]["pairs"][k])
            for u, v in zip(other["diff"], res[0]["diff"]):
                assert sorted(zip(*[a.tolist() for a in u])) == sorted(zip(*[a.tolist() for a in v]))
            assert sorted(other["due"].tolist()) == sorted(res[0]["due"].tolist())
            for k in ("vis", "cells"):
                for u, v in zip(other[k], res[0][k]):
                    np.testing.assert_array_equal(u, v)
            for u, v in zip(other["ho"], res[0]["ho"]):
                np.testing.assert_array_equal(np.sort(u), np.sort(v))
    assert engines[1].launch_count() == engines[2].launch_count()
    assert engines[0].launch_count() > engines[2].launch_count()


def test_delta_graph_replay_matches_direct_launches(chd):
    wc, x, z, idx, r = _world(chd, "benchmark", 30_000, 3_000)
    S = wc.n_subscribers
    engines = [chd.engine.Engine(wc.cfg(), wc.n_entities, S) for _ in range(2)]
    for e, on in zip(engines, (False, True)):
        e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
        e.reserve_visible_delta(1 << 20)
        e.enable_graphs(on)
    for t in range(8):
        x, z = chd.synth.move_entities(wc, x, z, t, 60.0)
        batch, keep = _batch(chd, idx, x, z, r)
        got = []
        for e in engines:
            e.set_entities(x, z)
            e.tick(batch, t * 33 * MS, chd.capi.TICK_BUILD | chd.capi.TICK_EMIT | chd.capi.TICK_VISIBLE_DELTA)
            got.append(e.get_visible_delta())
        for u, v in zip(*got):
            np.testing.assert_array_equal(u, v)
    assert engines[0].graph_launch_count() == 0 and engines[1].graph_launch_count() > 0
    # the delta stage on its own (no other stage runs): every call after the first sighting of its shape is a graph replay
    g0 = engines[1].graph_launch_count()
    for _ in range(4):
        got = []
        for e in engines:
            e.visible_delta()
            got.append(e.get_visible_delta())
        for u, v in zip(*got):
            np.testing.assert_array_equal(u, v)
        assert len(got[1][1]) == 0 and len(got[1][3]) == 0  # nothing changed since the last delta
    assert engines[0].graph_launch_count() == 0 and engines[1].graph_launch_count() - g0 >= 3


@pytest.mark.parametrize("mode", ["sync", "async"])
def test_delta_overflow_is_reported_by_the_early_read_back(chd, mode):
    """TICK_ALL | EARLY_RESULTS | VISIBLE_DELTA with chd_fetch_results / chd_fetch_results_async: CHD_OVF_DELTA is in the summary
    of the tick whose delta overflowed (the read-back of the counters waits for the delta), not in the next tick's."""
    import torch

    wc, x, z, idx, r = _world(chd, "benchmark", 200_000, 20_000)
    S = wc.n_subscribers
    L = chd.capi.lib()
    e = chd.engine.Engine(wc.cfg(), wc.n_entities, S, max_visible=1 << 25)
    e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
    e.reserve_visible_delta(10)  # the first delta enters every visible list: far more than 10 entries
    cap = 1 << 18
    due_t = torch.zeros(cap * 12, dtype=torch.int32).pin_memory()
    voff_t = torch.zeros(S + 1, dtype=torch.int64).pin_memory()
    hdr_t = torch.zeros(64, dtype=torch.int32).pin_memory()
    rb = chd.capi.ResultBuffers()
    rb.due, rb.due_cap = chd.capi.ptr(due_t), cap
    rb.vis_off = chd.capi.ptr(voff_t)
    ring_state = None
    for t in range(2):
        x, z = chd.synth.move_entities(wc, x, z, t, 60.0)
        ring_state, off, arr, snd, ridx, cmi = chd.synth.update_rings(wc, t, (t + 1) * 33 * MS, 33 * MS, 4, S, ring_len=16, state=ring_state)
        e.set_entities(x, z)
        e.set_rings(off, arr, snd, ridx, cmi)
        batch, keep = _batch(chd, idx, x, z, r)
        e.tick(batch, (t + 1) * 33 * MS, chd.capi.TICK_ALL | chd.capi.TICK_EARLY_RESULTS | chd.capi.TICK_VISIBLE_DELTA, want_summary=False)
        s = chd.capi.TickSummary()
        if mode == "sync":
            st = L.chd_fetch_results(e.h, C.byref(rb), C.byref(s))
        else:
            assert L.chd_fetch_results_async(e.h, C.byref(rb), chd.capi.ptr(hdr_t)) == chd.capi.OK
            st = L.chd_fetch_wait(e.h, C.byref(s))
        if t == 0:
            assert st == chd.capi.ERR_CAPACITY and s.overflow == chd.capi.OVF_DELTA
            ne, nl, _ = e.visible_delta_counts()
            assert ne == s.n_visible and nl == 0  # the required sizes
            e.reserve_visible_delta(1 << 25)
        else:
            assert st == chd.capi.OK and s.overflow == 0
            np.testing.assert_array_equal(voff_t.numpy().view(np.uint64), e.get_visible()[0])
            # the snapshot did not move at tick 0: this delta enters the full lists of tick 1
            _assert_delta(e.get_visible_delta(), _set_diff(EMPTY, e.get_visible(), S))


def test_delta_through_the_controller(chd):
    """GpuStaticGrid2DSpatialController: ReserveVisibleDelta, Tick with the flag, GetVisibleDelta = the set difference of the
    visible lists (reading the delta back never discards it)."""
    wc, x, z, idx, r = _world(chd, "benchmark", 30_000, 3_000)
    S = wc.n_subscribers
    c = chd.controller.GpuStaticGrid2DSpatialController(max_entities=wc.n_entities, max_subscribers=S)
    c.LoadConfig(dict(WorldOffsetX=wc.offx, WorldOffsetZ=wc.offz, GridWidth=wc.w, GridHeight=wc.h, GridCols=wc.cols, GridRows=wc.rows,
                      ServerCols=wc.server_cols, ServerRows=wc.server_rows))
    c.engine.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
    c.ReserveVisibleDelta(1 << 20)
    prev = EMPTY
    for t in range(3):
        x, z = chd.synth.move_entities(wc, x, z, t, 100.0)
        c.engine.set_entities(x, z)
        batch, keep = _batch(chd, idx, x, z, r)
        c.Tick(batch, t * 33 * MS, chd.capi.TICK_BUILD | chd.capi.TICK_EMIT | chd.capi.TICK_VISIBLE_DELTA)
        now = c.engine.get_visible()
        want = _set_diff(prev, now, S)
        _assert_delta(c.GetVisibleDelta(), want)
        _assert_delta(c.GetVisibleDelta(), want)  # a second read returns the same delta
        prev = now
