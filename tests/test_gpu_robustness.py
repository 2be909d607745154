"""GPU tests of the capacity / error rules of the C ABI (include/chd_gpu.h, CHD_OVF_*): an overflow or a malformed
query never corrupts the engine's state.  Findings of the round-1 review, each reproduced here."""
import ctypes as C

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
    from channeld_b200 import capi, engine, synth

    capi.lib()

    class NS:
        pass

    ns = NS()
    ns.capi, ns.engine, ns.synth = capi, engine, synth
    return ns


def _small_world(chd, n_sub=64, **lim):
    """8x8 grid of 100x100 cells at the origin; n_sub subscribers with sphere AOIs."""
    cfg = chd.engine.grid_cfg(0, 0, 100, 100, 8, 8)
    e = chd.engine.Engine(cfg, 1024, n_sub, **lim)
    rng = np.random.default_rng(7)
    ex, ez = rng.uniform(0, 800, 1000), rng.uniform(0, 800, 1000)
    e.set_entities(ex, ez)
    e.set_subscribers(np.arange(1, n_sub + 1, dtype=np.uint32))
    return e, rng


def _state(e):
    p = e.get_pairs()
    return {k: v.copy() for k, v in p.items()}


def _same_state(a, b):
    """Subscriptions and fan-out state equal (PF_NEW only says whether the LAST update created the pair)."""
    def norm(k, v):
        return v & ~np.uint8(2) if k == "flags" else v
    return all(np.array_equal(norm(k, a[k]), norm(k, b[k])) for k in a)


def test_window_overflow_leaves_state_untouched(chd):
    """A few huge AOIs exhaust max_window_cells: those queries fail with CHD_Q_ERR_CAPACITY, their subscribers keep their
    subscriptions, everybody else is updated, nothing is written out of bounds (review finding: chd_query.cuh OVF_WINDOW)."""
    capi = chd.capi
    n = 64
    e, rng = _small_world(chd, n, max_window_cells=320)
    cx, cz = rng.uniform(150, 650, n), rng.uniform(150, 650, n)
    r = np.full(n, 30.0)
    b, keep = chd.engine.make_batch(n, sphere=(cx, cz, r))
    s = e.tick(b, 1 * MS)
    assert s.overflow == 0 and s.n_query_errors == 0
    before = _state(e)
    # second update: small moves for everybody, but the last 8 subscribers ask for the whole world (64 cells each: only the
    # first one or two of them can still fit the 320-cell scratch once the small windows are placed)
    cx2, cz2 = cx + 40.0, cz + 40.0
    r2 = r.copy()
    r2[-8:] = 2000.0
    b2, keep2 = chd.engine.make_batch(n, sphere=(cx2, cz2, r2))
    with pytest.raises(chd.capi.ChdError) as ei:
        e.tick(b2, 2 * MS)
    assert ei.value.status == capi.ERR_CAPACITY
    st = e.get_query_status(n)
    failed = np.nonzero(st == capi.Q_ERR_CAPACITY)[0]
    assert len(failed) >= 1 and set(st.tolist()) <= {capi.Q_OK, capi.Q_ERR_CAPACITY}
    after = _state(e)
    want_status, want_off, want_id, want_dist = e.query_channel_ids(chd.engine.make_batch(n, sphere=(cx2, cz2, np.full(n, 30.0)))[0])
    for j in range(n):
        got = after["channel"][after["off"][j]:after["off"][j + 1]]
        if st[j] == capi.Q_ERR_CAPACITY:  # untouched
            np.testing.assert_array_equal(got, before["channel"][before["off"][j]:before["off"][j + 1]])
        elif r2[j] == 30.0:  # applied
            np.testing.assert_array_equal(got, want_id[want_off[j]:want_off[j + 1]])
    # the engine keeps working: a third, sane update is applied in full
    s3 = e.tick(b, 3 * MS)
    assert s3.overflow == 0 and s3.n_query_errors == 0
    assert _same_state({k: v for k, v in _state(e).items() if k in ("off", "channel", "dist")},
                       {k: v for k, v in before.items() if k in ("off", "channel", "dist")})
    e.close()


def test_pair_overflow_is_transactional(chd):
    """An interest update whose pair total exceeds max_pairs is not applied at all (review finding: the pair buffers were
    flipped over garbage)."""
    capi = chd.capi
    n = 64
    e, rng = _small_world(chd, n, max_pairs=200, max_window_cells=1 << 16)
    cx, cz = rng.uniform(150, 650, n), rng.uniform(150, 650, n)
    b, keep = chd.engine.make_batch(n, sphere=(cx, cz, np.full(n, 30.0)))
    s = e.tick(b, 1 * MS)
    assert s.overflow == 0 and s.n_pairs <= 200
    before = _state(e)
    big, keep2 = chd.engine.make_batch(n, sphere=(cx, cz, np.full(n, 400.0)))  # dozens of cells each: thousands of pairs
    with pytest.raises(chd.capi.ChdError) as ei:
        e.tick(big, 2 * MS)
    assert ei.value.status == capi.ERR_CAPACITY
    s2 = chd.capi.TickSummary()
    e.L.chd_summary(e.h, C.byref(s2))
    assert _same_state(_state(e), before)
    # the next sane update diffs against the untouched state: everything is "kept"
    s3 = e.tick(b, 3 * MS)
    assert s3.overflow == 0 and s3.n_kept == s3.n_pairs == s.n_pairs and s3.n_sub_new == 0 and s3.n_unsub == 0
    e.close()


def test_due_overflow_is_transactional(chd, oracle):
    """Decisions that do not fit max_due are neither delivered nor committed: the pairs stay due and catch up at the next
    tick (review finding: fan-out state was committed for dropped decisions)."""
    capi = chd.capi
    n = 64
    e, rng = _small_world(chd, n, max_due=16)
    cx, cz = rng.uniform(150, 650, n), rng.uniform(150, 650, n)
    b, keep = chd.engine.make_batch(n, sphere=(cx, cz, np.full(n, 30.0)))
    cells = 64
    e.set_rings(np.zeros(cells + 1, np.uint32), np.zeros(0, np.int64), np.zeros(0, np.uint32), np.zeros(0, np.uint64))
    s = e.tick(b, 0)
    P = int(s.n_pairs)
    assert P > 16
    # 100 ms later every pair is due for its first (FULL) fan-out: P decisions, capacity 16
    with pytest.raises(chd.capi.ChdError) as ei:
        e.tick(None, 100 * MS, capi.TICK_FANOUT)
    assert ei.value.status == capi.ERR_CAPACITY
    st = _state(e)
    had = (st["flags"] & capi.PF_HAD_FIRST) != 0
    due = e.get_due(16)
    real = due[due["kind"] != capi.DUE_VOID]
    assert had.sum() == len(real) <= 16 and (real["kind"] == 0).all()
    # every later tick delivers up to 16 more; nothing is lost, nothing is delivered twice
    delivered = set(zip(real["sub"].tolist(), real["channel_id"].tolist()))
    t = 100 * MS
    for _ in range(P):
        if len(delivered) == P:
            break
        t += 1 * MS
        try:
            s = e.tick(None, t, capi.TICK_FANOUT)
            n_due = s.n_due
        except chd.capi.ChdError as ex:
            assert ex.status == capi.ERR_CAPACITY
            n_due = 16
        due = e.get_due(min(n_due, 16))
        real = due[due["kind"] == 0]
        new = set(zip(real["sub"].tolist(), real["channel_id"].tolist()))
        assert not (new & delivered)
        delivered |= new
    assert len(delivered) == P
    e.close()


def test_missing_kind_arrays_are_a_query_error(chd):
    """A kind bit without its arrays is a per-query error, not a null dereference on the device."""
    capi = chd.capi
    e, rng = _small_world(chd, 4)
    kind = np.array([capi.AOI_SPHERE, capi.AOI_BOX, capi.AOI_SPHERE | capi.AOI_CONE, capi.AOI_SPHERE], np.uint8)
    b, keep = chd.engine.make_batch(4, kind=kind, sphere=(np.full(4, 400.0), np.full(4, 400.0), np.full(4, 30.0)))
    status, off, ids, dist = e.query_channel_ids(b)
    assert status.tolist() == [capi.Q_OK, capi.Q_ERR_MISSING_ARRAY, capi.Q_ERR_MISSING_ARRAY, capi.Q_OK]
    assert off[1] == off[2] == off[3] and off[4] > off[3]
    e.close()


def test_stateless_queries_do_not_disturb_interest_statuses(chd):
    capi = chd.capi
    e, rng = _small_world(chd, 4)
    cx = np.array([400.0, -50.0, 400.0, 400.0])  # query 1: centre out of the world
    b, keep = chd.engine.make_batch(4, sphere=(cx, np.full(4, 400.0), np.full(4, 30.0)))
    e.tick(b, 1 * MS)
    want = e.get_query_status(4).copy()
    assert want[1] == capi.Q_ERR_OUT_OF_WORLD
    ok, keep2 = chd.engine.make_batch(4, sphere=(np.full(4, 100.0), np.full(4, 100.0), np.full(4, 10.0)))
    st, *_ = e.query_channel_ids(ok)
    assert (st == 0).all()
    np.testing.assert_array_equal(e.get_query_status(4), want)
    e.close()


def test_cell_of_valid_with_id_start_zero(chd):
    cfg = chd.engine.grid_cfg(0, 0, 10, 10, 4, 4, id_start=0)
    e = chd.engine.Engine(cfg, 16, 4)
    ids, ok = e.cell_of(np.array([5.0, -1.0, 35.0]), np.array([5.0, 5.0, 35.0]), with_valid=True)
    assert ids.tolist() == [0, 0, 15] and ok.tolist() == [True, False, True]
    e.close()


def test_iteration_guards_match_the_oracle(chd, oracle):
    """Absorbed steps and oversized walks are rejected identically on both sides; |angle| >= 2^29 likewise."""
    from tests._oracle import make_grid

    capi = chd.capi
    cfg = chd.engine.grid_cfg(-1e6, -1e6, 20, 20, 100, 100)
    e = chd.engine.Engine(cfg, 16, 8)
    og = make_grid(-1e6, -1e6, 20, 20, 100, 100, 1, 1)
    cases = [
        dict(sphere=(1e17, 0.0, 5.0)),         # x + 2.5 == x: absorbed
        dict(sphere=(0.0, -3e18, 1.0)),        # z absorbed
        dict(sphere=(0.0, 0.0, 45000.0)),      # 4500^2 = 2e7 samples > 2^24
        dict(sphere=(0.0, 0.0, 20000.0)),      # 1.6e7 samples < 2^24: walked to the end (centre outside the world)
        dict(cone=(-999000.0, -999000.0, 1.0, 0.0, float(1 << 29), 50.0)),
        dict(cone=(-999000.0, -999000.0, 1.0, 0.0, float((1 << 29) - 1), 50.0)),
    ]
    for c in cases:
        if "sphere" in c:
            cx, cz, r = c["sphere"]
            b, keep = chd.engine.make_batch(1, sphere=(np.array([cx]), np.array([cz]), np.array([r])))
            want, wst = oracle.query(og, sphere=(cx, cz, r))
        else:
            cx, cz, dx, dz, ang, r = c["cone"]
            b, keep = chd.engine.make_batch(1, kind=np.array([capi.AOI_CONE], np.uint8),
                                            cone=tuple(np.array([v]) for v in (cx, cz, dx, dz, ang, r)))
            want, wst = oracle.query(og, cone=(cx, cz, dx, dz, ang, r))
        st, off, ids, dist = e.query_channel_ids(b, cap=1 << 16)
        assert int(st[0]) == int(wst), (c, st, wst)
        if wst == 0:
            assert dict(zip(ids.tolist(), dist.tolist())) == want
    e.close()


def test_subscriber_churn_parity(chd, oracle):
    """chd_add_subscribers / chd_remove_subscribers over 12 ticks of moving subscribers: the removed slots' subscriptions come
    back as unsub entries (UnsubscribeFromChannel, subscription.go:104-125), re-used slots start afresh, and the fan-out state of
    every OTHER pair stays bit-identical to the literal tickData emulation (one oracle channel per cell) — the round-1 engine
    could only reset everybody (chd_set_subscribers)."""
    from tests._oracle import make_grid

    g = (-300.0, -250.0, 100.0, 100.0, 6, 5)
    og = make_grid(*g)
    rng = np.random.default_rng(2024)
    S, N = 48, 300
    e = chd.engine.Engine(chd.engine.grid_cfg(*g), N, S + 16, max_visible=1 << 20)
    conn = np.zeros(S + 16, np.uint32)
    conn[:S] = np.arange(101, 101 + S)
    e.set_subscribers(conn[:S])
    e.set_entities(rng.uniform(-300, 300, N), rng.uniform(-250, 250, N))
    e.build()
    cells = g[4] * g[5]
    chans = [oracle.channel() for _ in range(cells)]
    rings = [[] for _ in range(cells)]
    msg_index = np.zeros(cells, np.uint64)
    n_slots = S + 16
    cx, cz = rng.uniform(-280, 280, n_slots), rng.uniform(-230, 230, n_slots)
    rad = rng.choice([30.0, 60.0, 120.0], n_slots)
    active = np.zeros(n_slots, bool)
    active[:S] = True
    subs_now = [dict() for _ in range(n_slots)]
    next_conn = 1000
    t = 0
    seen_removed = seen_added = 0
    for tick in range(12):
        t += 33 * MS if tick % 3 else 80 * MS
        cx += rng.uniform(-40, 40, n_slots)
        cz += rng.uniform(-40, 40, n_slots)
        # ---- churn before the update: some connections close, some new ones arrive (into free slots, incl. ones beyond S)
        want_un = set()
        if tick >= 2:
            leave = rng.choice(np.nonzero(active)[0], size=int(rng.integers(1, 5)), replace=False)
            e.remove_subscribers(leave)
            for j in leave:
                for c in list(subs_now[j].keys()):
                    want_un.add((int(j), int(c)))
                    chans[c - S0].unsubscribe(int(conn[j]))
                subs_now[j].clear()
                active[j] = False
                seen_removed += 1
            free = np.nonzero(~active)[0]
            free = free[~np.isin(free, leave)]  # a slot removed this tick is free only after the update
            join = rng.choice(free, size=min(len(free), int(rng.integers(0, 4))), replace=False)
            if len(join):
                ids = np.arange(next_conn, next_conn + len(join), dtype=np.uint32)
                next_conn += len(join)
                e.add_subscribers(join, ids)
                conn[join] = ids
                active[join] = True
                seen_added += len(join)
        else:
            leave = np.zeros(0, np.int64)
        moving = active & (rng.random(n_slots) < 0.8)
        qi = np.nonzero(moving | np.isin(np.arange(n_slots), leave))[0].astype(np.uint32)  # removed slots' queries are ignored
        batch, keep = chd.engine.make_batch(len(qi), sub=qi, sphere=(cx[qi], cz[qi], rad[qi]))
        e.update_interest(batch, t)
        s = e.summary()
        (new_s, new_c), (un_s, un_c) = e.get_diff(s.n_sub_new, s.n_unsub)
        want_new = set()
        for j in qi:
            if not moving[j]:
                continue
            res, st = oracle.query(og, sphere=(cx[j], cz[j], rad[j]))
            if st != 0:
                continue
            un, sn, kp = oracle.interest_diff(list(subs_now[j].keys()), list(res.keys()))
            for c in un:
                want_un.add((int(j), int(c)))
                chans[c - S0].unsubscribe(int(conn[j]))
                del subs_now[j][int(c)]
            for c in list(sn) + list(kp):
                chans[c - S0].subscribe(int(conn[j]), t, oracle.damping(res[int(c)], 20), 0, True, False)
                subs_now[j][int(c)] = res[int(c)]
            want_new |= {(int(j), int(c)) for c in sn}
        assert set(zip(new_s.tolist(), new_c.tolist())) == want_new
        assert set(zip(un_s.tolist(), un_c.tolist())) == want_un
        pairs = e.get_pairs()
        assert len(pairs["off"]) == e.n_slots + 1
        for j in range(e.n_slots):
            sl = slice(pairs["off"][j], pairs["off"][j + 1])
            assert dict(zip(pairs["channel"][sl].tolist(), pairs["dist"][sl].tolist())) == subs_now[j], (tick, j)
        # ---- updates + fan-out
        for _ in range(int(rng.integers(5, 30))):
            c = int(rng.integers(0, cells))
            arrival = t - int(rng.integers(0, 60)) * MS
            sender = int(rng.choice(conn[active])) if rng.random() < 0.5 else 7
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
        want = []
        for c in range(cells):
            for d in chans[c].tick_data_ex(t):
                want.append((d["conn"], S0 + c, d["kind"], d["n"], d["first"], d["last"], d["hash"], d["last_index"], d["window_hi"]))
        got = [(int(conn[d["sub"]]), int(d["channel_id"]), int(d["kind"]), int(d["n_selected"]), int(d["first_sel"]), int(d["last_sel"]),
                int(d["sel_hash"]), int(d["last_message_index"]), int(d["window_hi"])) for d in due]
        assert sorted(got) == sorted(want), tick
        pairs = e.get_pairs()
        for j in range(e.n_slots):
            for p in range(pairs["off"][j], pairs["off"][j + 1]):
                last, had, idx = chans[int(pairs["channel"][p]) - S0].state(int(conn[j]))
                assert (int(pairs["last"][p]), bool(pairs["flags"][p] & 1), int(pairs["last_index"][p])) == (last, had, idx), (tick, j)
    assert seen_removed >= 10 and seen_added >= 5
    e.close()


def test_device_owned_rings_and_channel_time_origins(chd, oracle):
    """ChannelData.OnUpdate's buffer on the device (chd_rings_init / chd_rings_append, data.go:149-173) incl. the > 512 eviction
    rule with the device-tracked maxFanOutIntervalMs, and per-channel ChannelTime origins (channel.go:178): ring contents,
    message indices and every fan-out decision match one oracle channel per cell fed the same updates in its own clock."""
    from tests._oracle import make_grid

    capi = chd.capi
    g = (0.0, 0.0, 100.0, 100.0, 3, 2)
    og = make_grid(*g)
    cells = 6
    rng = np.random.default_rng(77)
    S = 24
    e = chd.engine.Engine(chd.engine.grid_cfg(*g), 64, S, max_ring_entries=cells * 1024)
    conn = np.arange(201, 201 + S, dtype=np.uint32)
    e.set_subscribers(conn)
    e.set_entities(rng.uniform(0, 300, 50), rng.uniform(0, 200, 50))
    e.build()
    start = rng.integers(0, 500, cells).astype(np.int64) * MS  # every channel was created at a different wall time
    assert e.L.chd_set_channel_start_times(e.h, capi.ptr(start)) == capi.OK
    assert e.L.chd_rings_init(e.h, 1024) == capi.OK
    # host-owned rings cannot be prefetched over device-owned ones: a short set (one entry) is refused, so nothing is staged
    # and the device-owned rings keep all their entries (checked against the oracle below)
    short_off = np.array([0] + [1] * cells, np.uint32)
    short_arr, short_snd, short_idx = np.array([1000 * MS], np.int64), np.array([7], np.uint32), np.array([1], np.uint64)
    assert e.L.chd_prefetch_rings(e.h, capi.ptr(short_off), 1, capi.ptr(short_arr), capi.ptr(short_snd), capi.ptr(short_idx), None) == capi.ERR_STATE
    assert e.L.chd_adopt_prefetched(e.h) == capi.ERR_STATE
    chans = [oracle.channel() for _ in range(cells)]
    cx, cz = rng.uniform(20, 280, S), rng.uniform(20, 180, S)
    rad = rng.choice([30.0, 80.0], S)
    t = 1000 * MS
    total_due = 0
    evicted = False
    for tick in range(14):
        t += 40 * MS
        cx = np.clip(cx + rng.uniform(-30, 30, S), 1, 299)
        cz = np.clip(cz + rng.uniform(-30, 30, S), 1, 199)
        batch, keep = chd.engine.make_batch(S, sphere=(cx, cz, rad))
        e.update_interest(batch, t)
        e.summary()
        for j in range(S):
            res, st = oracle.query(og, sphere=(cx[j], cz[j], rad[j]))
            assert st == 0
            for c in range(cells):
                if S0 + c in res:
                    chans[c].subscribe(int(conn[j]), t - int(start[c]), oracle.damping(res[S0 + c], 20), 0, True, False)
                else:
                    chans[c].unsubscribe(int(conn[j]))
        # updates of this tick, CSR by cell, in arrival order per cell; cell 0 gets a flood (buffer > 512 -> eviction rule)
        per_cell = [int(rng.integers(0, 6)) for _ in range(cells)]
        per_cell[0] = 120
        upd_off = np.concatenate([[0], np.cumsum(per_cell)]).astype(np.uint32)
        arr, snd = [], []
        for c in range(cells):
            ts = np.sort(rng.integers(0, 40, per_cell[c])) * MS + (t - 40 * MS) - int(start[c])  # channel time of channel c
            for a in ts:
                s_ = int(rng.choice(conn)) if rng.random() < 0.4 else 7
                arr.append(int(a)); snd.append(s_)
                chans[c].on_update(int(a), s_)
        arr_np, snd_np = np.array(arr, np.int64), np.array(snd, np.uint32)  # (named: a temporary could be freed before the call)
        st_ = e.L.chd_rings_append(e.h, capi.ptr(upd_off), len(arr), capi.ptr(arr_np), capi.ptr(snd_np))
        assert st_ == capi.OK, e.L.chd_last_error(e.h)
        # ring contents
        roff = np.zeros(cells + 1, np.uint32)
        ra, rs, ri = np.zeros(cells * 1024, np.int64), np.zeros(cells * 1024, np.uint32), np.zeros(cells * 1024, np.uint64)
        cmi = np.zeros(cells, np.uint64)
        st_ = e.L.chd_get_rings(e.h, capi.ptr(roff), capi.ptr(ra), capi.ptr(rs), capi.ptr(ri), capi.ptr(cmi), cells * 1024)
        assert st_ == capi.OK, e.L.chd_last_error(e.h)
        for c in range(cells):
            assert roff[c + 1] - roff[c] == chans[c].ring_len(), (tick, c)
        if roff[1] - roff[0] >= 512 and ri[roff[0]] > 1:
            evicted = True  # the head of cell 0's ring moved: entries older than maxFanOutIntervalMs left once the buffer passed 512
        e.fanout_tick(t)
        s = e.summary()
        assert s.overflow == 0
        due = e.get_due(s.n_due)
        want = []
        for c in range(cells):
            for d in chans[c].tick_data_ex(t - int(start[c])):
                want.append((d["conn"], S0 + c, d["kind"], d["n"], d["first"], d["last"], d["hash"], d["last_index"], d["window_hi"]))
        got = [(int(conn[d["sub"]]), int(d["channel_id"]), int(d["kind"]), int(d["n_selected"]), int(d["first_sel"]), int(d["last_sel"]),
                int(d["sel_hash"]), int(d["last_message_index"]), int(d["window_hi"])) for d in due]
        if sorted(got) != sorted(want):
            only_got, only_want = sorted(set(got) - set(want)), sorted(set(want) - set(got))
            c0 = only_got[0][1] - S0 if only_got else only_want[0][1] - S0
            ring_c = list(zip(ra[roff[c0]:roff[c0 + 1]].tolist(), rs[roff[c0]:roff[c0 + 1]].tolist(), ri[roff[c0]:roff[c0 + 1]].tolist()))
            raise AssertionError("tick %d start[c]=%d only_got=%r only_want=%r ring[%d][235:250]=%r" % (tick, int(start[c0]), only_got[:6], only_want[:6], c0, ring_c[235:250]))
        total_due += len(got)
        pairs = e.get_pairs()
        for j in range(S):
            for p in range(pairs["off"][j], pairs["off"][j + 1]):
                last, had, idx = chans[int(pairs["channel"][p]) - S0].state(int(conn[j]))
                assert (int(pairs["last"][p]), bool(pairs["flags"][p] & 1), int(pairs["last_index"][p])) == (last, had, idx), (tick, j)
    assert total_due > 100 and evicted
    e.close()
