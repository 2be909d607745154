"""The two-stream tick leaves its visible-list copy kernel running on the copy stream: the next tick's build, interest update and
emit preparation run beside it, writing the other of the two copy-input sets.  Each case compares an engine driven back to back,
with no host sync between ticks, against one that calls chd_summary after every tick (the drained engine).  With a single set
of copy inputs, the next head would rewrite what the copy still reads, and these comparisons would fail.

Two worlds, on each side of the host's kernel choice (CTA tiles and warp tiles, shapes as in test_gpu_emit_order.py), plus
entity-table mode.
Run on an H100:  python -m pytest tests -m gpu
"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SENTINEL = 0xDEADBEEF
# (grid: offset, cell size, cols, rows), entities, subscribers, radii
WORLDS = {
    "cta": ((-4000.0, 2000.0, 4, 4), 24_000, 2_000, (50.0, 1500.0)),
    "warp": ((-800.0, 100.0, 16, 16), 38_400, 4_000, (20.0, 120.0)),
}


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
    ns.torch, ns.capi, ns.engine, ns.synth = torch, capi, engine, synth
    return ns


class _DeviceArray:
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i4", "data": (ptr, False), "version": 3}


def _vis_tensor(chd, e):
    ptr, n = e.device_view(chd.capi.VIEW_VIS_ENTITY)
    return chd.torch.as_tensor(_DeviceArray(ptr, n), device="cuda")


def _vis(chd, e, n):
    return _vis_tensor(chd, e)[:n].cpu().numpy().view(np.uint32).copy()


def _fill_visible(chd, e):
    _vis_tensor(chd, e).fill_(SENTINEL - (1 << 32))
    chd.torch.cuda.synchronize()


def _world(chd, name, table=False):
    (off, size, cols, rows), n, n_sub, (r_lo, r_hi) = WORLDS[name]
    wc = chd.synth.WorldConfig("pipeline-" + name, off, off, size, size, cols, rows, 1, 1, n, n_sub, r_lo, 31)
    ex, ez = chd.synth.entities(wc)
    rng = np.random.default_rng(7)
    stand = rng.integers(0, n, n_sub)
    cx, cz = ex[stand].copy(), ez[stand].copy()
    r = rng.uniform(r_lo, r_hi, n_sub)
    frames = []
    for k in range(6):  # moving entities, alternating large and small radii
        x, z = chd.synth.move_entities(wc, ex, ez, k, size * 0.05)
        frames.append((x.copy(), z.copy(), r * (3.0 if k % 2 == 0 else 1.0)))
    return wc, (cx, cz), frames


def _engine(chd, wc, table):
    e = chd.engine.Engine(wc.cfg(), wc.n_entities, wc.n_subscribers, max_visible=1 << 26, max_pairs=1 << 20, max_window_cells=1 << 22)
    e.set_subscribers(np.arange(1, wc.n_subscribers + 1, dtype=np.uint32))
    if table:
        e.entity_table_init()
    return e


def _set_positions(e, table, x, z):
    if table:
        ids = np.arange(1000, 1000 + len(x), dtype=np.uint32)
        if not getattr(e, "_spawned", False):
            e.spawn_entities(ids, x, z)
            e._spawned = True
        else:
            e.move_entities(ids, x, z)
    else:
        e.set_entities(x, z)


def _tick(chd, e, q, f, k, flags, summary):
    batch, keep = chd.engine.make_batch(len(q[0]), sub=None, sphere=(q[0], q[1], f[2]))
    e._keep_batch = (batch, keep)
    return e.tick(batch, (k + 1) * 33_000_000, flags, want_summary=summary)


CASES = [("cta", False), ("warp", False), ("cta", True)]
IDS = ["cta", "warp", "cta-table"]


@pytest.mark.parametrize("name,table", CASES, ids=IDS)
def test_copy_beside_the_next_head_keeps_both_lists(chd, name, table):
    """A large-radius tick then a small-radius one, back to back.  After draining, [0, V_small) holds the small tick's lists and
    [V_small, V_large) still holds what the large tick's copy wrote while build, interest and preparation of the small tick ran."""
    wc, q, frames = _world(chd, name)
    flags = chd.capi.TICK_BUILD | chd.capi.TICK_EMIT
    ref = _engine(chd, wc, table)
    _fill_visible(chd, ref)
    want = []
    for k in range(2):
        _set_positions(ref, table, frames[k][0], frames[k][1])
        s = _tick(chd, ref, q, frames[k], k, flags, True)
        want.append((s.n_visible, _vis(chd, ref, s.n_visible)))
    ref.close()
    v_large, v_small = want[0][0], want[1][0]
    assert v_large > 2 * v_small > 0

    e = _engine(chd, wc, table)
    _fill_visible(chd, e)
    for k in range(2):
        _set_positions(e, table, frames[k][0], frames[k][1])
        _tick(chd, e, q, frames[k], k, flags, False)
    s = e.summary()
    assert s.n_visible == v_small and s.overflow == 0
    got = _vis(chd, e, v_large + 1024)
    np.testing.assert_array_equal(got[:v_small], want[1][1])
    np.testing.assert_array_equal(got[v_small:v_large], want[0][1][v_small:v_large])
    assert (got[v_large:v_large + 1024] == SENTINEL).all()
    e.close()


@pytest.mark.parametrize("name,table", CASES, ids=IDS)
def test_build_and_interest_beside_the_copy(chd, name, table):
    """A tick with CHD_TICK_EMIT, then one without it (build, fan-out and an interest update): the first tick's whole expanded
    list stays intact."""
    wc, q, frames = _world(chd, name)
    ref = _engine(chd, wc, table)
    _set_positions(ref, table, frames[0][0], frames[0][1])
    s0 = _tick(chd, ref, q, frames[0], 0, chd.capi.TICK_BUILD | chd.capi.TICK_EMIT, True)
    want = _vis(chd, ref, s0.n_visible)
    ref.close()

    e = _engine(chd, wc, table)
    _set_positions(e, table, frames[0][0], frames[0][1])
    _tick(chd, e, q, frames[0], 0, chd.capi.TICK_BUILD | chd.capi.TICK_EMIT, False)
    _set_positions(e, table, frames[1][0], frames[1][1])
    _tick(chd, e, q, frames[1], 1, chd.capi.TICK_BUILD | chd.capi.TICK_FANOUT, False)
    e.summary()
    np.testing.assert_array_equal(_vis(chd, e, len(want)), want)
    e.close()


@pytest.mark.parametrize("name,table", CASES, ids=IDS)
def test_documented_calls_wait_for_the_copy(chd, name, table):
    """Right after chd_tick, with no summary: chd_get_visible_slot, and a torch read of chd_device_view(CHD_VIEW_VIS_ENTITY) on
    the engine stream, see the tick's final expanded list."""
    wc, q, frames = _world(chd, name)
    flags = chd.capi.TICK_BUILD | chd.capi.TICK_EMIT
    ref = _engine(chd, wc, table)
    for k in range(3):
        _set_positions(ref, table, frames[k][0], frames[k][1])
        s = _tick(chd, ref, q, frames[k], k, flags, True)
    want = _vis(chd, ref, s.n_visible)
    voff, _ = ref.get_visible()
    slot = int(np.argmax(np.diff(voff)))
    ref.close()

    torch = chd.torch
    stream = torch.cuda.Stream()
    for view in (False, True):
        e = _engine(chd, wc, table)
        e.set_stream(stream.cuda_stream)
        for k in range(3):
            _set_positions(e, table, frames[k][0], frames[k][1])
            _tick(chd, e, q, frames[k], k, flags, False)
        if view:
            t = _vis_tensor(chd, e)
            with torch.cuda.stream(stream):
                got = t[:len(want)].clone()
            stream.synchronize()
            np.testing.assert_array_equal(got.cpu().numpy().view(np.uint32), want)
        else:
            lst = e.get_visible_slot(slot)
            np.testing.assert_array_equal(lst, want[voff[slot]:voff[slot + 1]])
        e.close()


@pytest.mark.parametrize("name,table", CASES, ids=IDS)
def test_async_results_of_every_tick_match_the_drained_engine(chd, name, table):
    """Six ticks back to back with changing positions and alternating radii, each tick's results read with
    chd_fetch_results_async / chd_fetch_wait while the next one runs: pairs, diff, handover, cell CSR, statuses and visible
    offsets equal a drained engine's getters."""
    torch = chd.torch
    wc, q, frames = _world(chd, name)
    S, cap = wc.n_subscribers, 1 << 20
    flags = chd.capi.TICK_BUILD | chd.capi.TICK_EMIT

    ref = _engine(chd, wc, table)
    want = []
    for k, f in enumerate(frames):
        _set_positions(ref, table, f[0], f[1])
        s = _tick(chd, ref, q, f, k, flags, True)
        voff, _ = ref.get_visible()
        cs, se = ref.get_cells()
        want.append(dict(s=s.as_dict(), pairs=ref.get_pairs(s.n_pairs), diff=ref.get_diff(s.n_sub_new, s.n_unsub),
                         ho=ref.get_handover(s.n_handover), st=ref.get_query_status(S), voff=voff, cs=cs, se=se))
    ref.close()

    def pin(n, dt):
        t_ = torch.zeros(n, dtype=dt).pin_memory()
        return t_, t_.numpy()

    def result_set():
        k = {n_: pin(cap, torch.int32) for n_ in ("ch", "dist", "iv", "ns", "nc", "us", "uc", "he", "hs", "hd", "st", "se")}
        k["off"], k["voff"], k["cs"] = pin(S + 1, torch.int32), pin(S + 1, torch.int64), pin(wc.cells + 1, torch.int32)
        k["hdr"] = pin(64, torch.int32)
        rb = chd.capi.ResultBuffers()
        P = lambda n_: chd.capi.ptr(k[n_][0])  # noqa: E731
        rb.pair_off, rb.pair_channel, rb.pair_dist, rb.pair_interval_ms, rb.pair_cap = P("off"), P("ch"), P("dist"), P("iv"), cap
        rb.new_sub, rb.new_channel, rb.unsub_sub, rb.unsub_channel, rb.diff_cap = P("ns"), P("nc"), P("us"), P("uc"), cap
        rb.handover_entity, rb.handover_src, rb.handover_dst, rb.handover_cap = P("he"), P("hs"), P("hd"), cap
        rb.query_status, rb.status_cap = P("st"), cap
        rb.vis_off, rb.vis_entity, rb.vis_cap = P("voff"), None, 0
        rb.cell_start, rb.sorted_entity, rb.entity_cap = P("cs"), P("se"), cap
        return rb, k

    def check(i, s, k):
        w = want[i]
        assert s.as_dict() == w["s"], i
        n = s.n_pairs
        np.testing.assert_array_equal(k["off"][1].view(np.uint32), w["pairs"]["off"])
        for a, b in (("ch", "channel"), ("dist", "dist"), ("iv", "interval")):
            np.testing.assert_array_equal(k[a][1][:n].view(np.uint32), w["pairs"][b])
        (a, b), (c, d) = w["diff"]
        canon = lambda u, v: np.sort(u.astype(np.uint64) << np.uint64(32) | v.astype(np.uint64))  # noqa: E731
        np.testing.assert_array_equal(canon(k["ns"][1][:s.n_sub_new].view(np.uint32), k["nc"][1][:s.n_sub_new].view(np.uint32)), canon(a, b))
        np.testing.assert_array_equal(canon(k["us"][1][:s.n_unsub].view(np.uint32), k["uc"][1][:s.n_unsub].view(np.uint32)), canon(c, d))
        ho_g = np.stack([k[a][1][:s.n_handover].view(np.uint32) for a in ("he", "hs", "hd")], 1)
        ho_w = np.stack(w["ho"], 1)
        srt = lambda h: h[np.lexsort((h[:, 2], h[:, 1], h[:, 0]))]  # noqa: E731
        np.testing.assert_array_equal(srt(ho_g), srt(ho_w))
        np.testing.assert_array_equal(k["st"][1][:S].view(np.uint32), w["st"])
        np.testing.assert_array_equal(k["voff"][1].view(np.uint64), w["voff"])
        np.testing.assert_array_equal(k["cs"][1].view(np.uint32), w["cs"])
        np.testing.assert_array_equal(k["se"][1][:s.n_entities_in_world].view(np.uint32), w["se"])

    e = _engine(chd, wc, table)
    sets = [result_set(), result_set()]
    s = chd.capi.TickSummary()
    for i, f in enumerate(frames):
        _set_positions(e, table, f[0], f[1])
        _tick(chd, e, q, f, i, flags, False)
        rb, k = sets[i % 2]
        e._ck(e.L.chd_fetch_results_async(e.h, C.byref(rb), chd.capi.ptr(k["hdr"][0])))
        if i:
            e._ck(e.L.chd_fetch_wait(e.h, C.byref(s)))
            check(i - 1, s, sets[(i - 1) % 2][1])
    e._ck(e.L.chd_fetch_wait(e.h, C.byref(s)))
    check(len(frames) - 1, s, sets[(len(frames) - 1) % 2][1])
    assert sum(w["s"]["n_handover"] for w in want) > 0
    e.close()
