"""Byte-carrying device rings (include/chd_gpu_ring_bytes.h) on sharded engines, in the world of tests/test_gpu_sharded_rings.py:
  slabs      2 and 3 slabs on one device (chd_set_slab, the host-joined ring-limit exchange), every rank appending the whole-grid
             updates with their bytes: every tick each rank's served rings and their bytes equal a whole-world byte-carrying engine's,
             and the class entry of each of its decisions equals the whole-world engine's entry for the same (connection, channel,
             kind, window_hi, last_message_index)
  world one  chd_tick_sharded on a one-rank communicator: the bytes chd_rings_append_bytes staged are applied by the tick (rings,
             bytes and class entries equal a plain engine's), assembling between ticks is accepted, and while updates are staged a
             second append, chd_get_ring_bytes and the reserve are refused, changing nothing and launching nothing
Run on an H100:  python -m pytest tests/test_ring_bytes_sharded_gpu.py -m gpu
"""
import numpy as np
import pytest

from tests.test_gpu_payload_scale import Payload
from tests.test_gpu_sharded_rings import (COLS, DEFAULT_IV, HALO, ROWS, W, RingWorld, _assert_rings_on, _batch, _compare, _due_set, _served,  # noqa: F401
                                          _world_one, chd)
from tests.test_ring_bytes_gpu import MAX_LEN, _append_bytes, _assert_bytes, _entries_by_decision

pytestmark = pytest.mark.gpu

CAP = 620


def _full(rng):
    f_len = rng.integers(0, 300, COLS * ROWS)
    off = np.concatenate([[0], np.cumsum(f_len)]).astype(np.uint64)
    return off, np.frombuffer(rng.bytes(int(off[-1])), np.uint8)


def _entries(pl, e, conn_of_slot, n_due, full):
    """the class entry of every decision of the last fan-out pass -> dict keyed by the decision's identity"""
    pl.set_bytes(np.zeros(1, np.uint64), np.zeros(0, np.uint8), *full)
    n_cls, cls_off, blob = pl.assemble()
    got, _ = _entries_by_decision(conn_of_slot, e, e.get_due(n_due), cls_off, blob)
    out = dict(got)
    assert len(out) == len(got)
    return out


@pytest.mark.parametrize("world", [2, 3])
def test_slab_replicas_carry_the_whole_world_bytes(chd, world):
    import torch

    rw = RingWorld(world, CAP, 41 + world)
    cfg = chd.engine.grid_cfg(0.0, 0.0, W, W, COLS, ROWS)
    conn_all = np.concatenate(rw.conn)
    whole = chd.engine.Engine(cfg, 16, len(conn_all), default_fanout_interval_ms=DEFAULT_IV)
    whole.set_subscribers(conn_all)
    engines, served = [], []
    for r in range(world):
        lo, hi = chd.sharding.slab_columns(COLS, world, r)
        e = chd.engine.Engine(cfg, 16, len(rw.conn[r]), default_fanout_interval_ms=DEFAULT_IV)
        e.set_slab(lo, hi, HALO)
        e.set_subscribers(rw.conn[r])
        engines.append(e)
        served.append(_served(lo, hi))
    for e in engines + [whole]:
        e.rings_init(CAP)
        e.rings_reserve_bytes(CAP * (MAX_LEN + 1))
    pls = [Payload(chd, e, len(rw.conn[r])) for r, e in enumerate(engines)]
    pw = Payload(chd, whole, len(conn_all))
    rng = np.random.default_rng(43)
    rec_cap = max(len(s) for s in served)
    recs = [torch.zeros(2 * rec_cap, dtype=torch.int32, device="cuda") for _ in range(world)]
    gathered, n_gathered = None, 0
    msg_before = np.zeros(COLS * ROWS, np.uint64)
    n_compared = n_update = 0
    for tick, t in enumerate(rw.times()):
        upd = rw.updates(tick, t)
        full = _full(rng)
        if n_gathered:
            for e in engines:
                e.import_ring_limits(gathered, n_gathered)
        whole._ck(_append_bytes(chd, whole, *upd, msg_before))
        sw = whole.tick(_batch(chd, *rw.queries(range(world), tick))[0], t, chd.capi.TICK_FANOUT)
        assert sw.overflow == 0
        W_rings = whole.get_rings()
        _assert_bytes(whole, W_rings)
        w_due = _due_set(whole, sw.n_due, conn_all)
        w_entries = _entries(pw, whole, conn_all, sw.n_due, full)
        for r, e in enumerate(engines):
            e._ck(_append_bytes(chd, e, *upd, msg_before))
            s = e.tick(_batch(chd, *rw.queries([r], tick))[0], t, chd.capi.TICK_FANOUT)
            assert s.overflow == 0
            got = e.get_rings()
            _assert_rings_on(got, W_rings, served[r], "tick %d rank %d" % (tick, r))
            _assert_bytes(e, got)  # every entry carries its own bytes; with the rings above, the served cells' bytes are the whole world's
            mine = set(rw.conn[r].tolist())
            assert _due_set(e, s.n_due, rw.conn[r]) == {x for x in w_due if x[0] in mine}, (tick, r)
            for key, entry in _entries(pls[r], e, rw.conn[r], s.n_due, full).items():
                assert entry == w_entries[key], (tick, r, key)
                n_compared += 1
                n_update += key[2] == 1
        msg_before = W_rings["msg_index"].copy()
        parts = []
        for r, e in enumerate(engines):
            k = e.export_ring_limits(recs[r], rec_cap)
            torch.cuda.synchronize()
            parts.append(recs[r][:2 * k].clone())
        gathered = torch.cat(parts)
        n_gathered = len(gathered) // 2
    for e in engines + [whole]:
        e.close()
    assert n_compared > 100 and n_update > 20


def _setup(chd, graphs):
    rw, sh, one, conn, x, z = _world_one(chd, graphs)
    for e in (sh, one):
        e.rings_reserve_bytes(CAP * (MAX_LEN + 1))
    return rw, sh, one, conn, x, z


def _refused(e, st, call):
    n = e.launch_count()
    assert call() == st
    assert e.launch_count() == n


@pytest.mark.parametrize("graphs", [True, False])
def test_tick_sharded_applies_the_staged_bytes(chd, graphs):
    capi = chd.capi
    rw, sh, one, conn, x, z = _setup(chd, graphs)
    rng = np.random.default_rng(47)
    psh, pone = Payload(chd, sh, len(conn)), Payload(chd, one, len(conn))
    msg_before = np.zeros(COLS * ROWS, np.uint64)
    n_update = 0
    for tick, t in enumerate(rw.times()[:6]):
        upd = rw.updates(tick, t)
        b, keep = _batch(chd, *rw.queries([0, 1], tick))
        sh.set_entities(x, z)
        sh.set_entity_ids(np.arange(len(x), dtype=np.uint32))
        one.set_entities(x, z)
        for e in (sh, one):
            assert _append_bytes(chd, e, *upd, msg_before) == capi.OK
        if tick == 1:  # rule 12: staged updates
            other = rw.updates(tick, t)
            _refused(sh, capi.ERR_STATE, lambda: _append_bytes(chd, sh, *other, msg_before))
            _refused(sh, capi.ERR_STATE, lambda: sh.L.chd_get_ring_bytes(sh.h, None, None, 0, None))
            assert "staged" in sh.L.chd_last_error(sh.h).decode()
            _refused(sh, capi.ERR_STATE, lambda: sh.L.chd_rings_reserve_bytes(sh.h, 64))
        s1 = sh.tick_sharded(b, t, capi.TICK_ALL)
        s2 = one.tick(b, t, capi.TICK_ALL)
        _compare(chd, sh, one, s1, s2, conn)
        rings = sh.get_rings()
        _assert_bytes(sh, rings)
        _assert_bytes(one, rings)
        msg_before = rings["msg_index"].copy()
        full = _full(rng)
        a, c = _entries(psh, sh, conn, s1.n_due, full), _entries(pone, one, conn, s2.n_due, full)  # between ticks: accepted
        assert a == c
        n_update += sum(k[2] == 1 for k in a)
    assert n_update > 20
    assert chd.capi.lib().chd_comm_destroy(sh.h) == capi.OK
    for e in (sh, one):
        e.close()


def test_reserve_is_refused_while_updates_are_staged(chd):
    """A staged append was checked against the byte slab it was staged for: until chd_tick_sharded applies it, the reserve is refused,
    also after a chd_rings_init, and the tick then applies the staged bytes to that slab."""
    capi = chd.capi
    rw, sh, one, conn, x, z = _world_one(chd, True)
    one.close()
    cells = COLS * ROWS
    # without the reservation: a staged chd_rings_append, chd_rings_init, then the reserve
    off = np.zeros(cells + 1, np.uint32)
    off[1:] = 1
    sh.rings_append(off, np.array([5], np.int64), np.array([3], np.uint32))
    sh.rings_init(CAP)
    _refused(sh, capi.ERR_STATE, lambda: sh.L.chd_rings_reserve_bytes(sh.h, 1000))
    t = rw.times()[0]
    b, keep = _batch(chd, *rw.queries([0, 1], 0))
    sh.set_entities(x, z)
    sh.set_entity_ids(np.arange(len(x), dtype=np.uint32))
    sh.tick_sharded(b, t, capi.TICK_ALL)
    assert chd.capi.lib().chd_comm_destroy(sh.h) == capi.OK
    sh.close()
    # with it: a staged 900-byte update, chd_rings_init, then a reserve of 100 bytes per cell
    rw, sh, one, conn, x, z = _world_one(chd, True)
    one.close()
    sh.rings_reserve_bytes(1000)
    boff = np.array([0, 900], np.uint64)
    data = (np.arange(900) % 251).astype(np.uint8)
    p = capi.ptr
    arr, snd = np.array([t - 1], np.int64), np.array([3], np.uint32)
    assert sh.L.chd_rings_append_bytes(sh.h, p(off), 1, p(arr), p(snd), p(boff), p(data)) == capi.OK
    sh.rings_init(CAP)
    _refused(sh, capi.ERR_STATE, lambda: sh.L.chd_rings_reserve_bytes(sh.h, 100))
    sh.set_entities(x, z)
    sh.set_entity_ids(np.arange(len(x), dtype=np.uint32))
    s = sh.tick_sharded(b, t, capi.TICK_ALL)
    assert s.overflow == 0
    rings = sh.get_rings()
    assert int(rings["off"][-1]) == 1 and int(rings["off"][1]) == 1
    got_off, got = sh.get_ring_bytes()
    assert got_off.tolist() == [0, 900] and got.tobytes() == data.tobytes()
    assert chd.capi.lib().chd_comm_destroy(sh.h) == capi.OK
    sh.close()
