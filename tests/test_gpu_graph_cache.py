"""The CUDA-graph cache of the launch-bound stages: every stage keeps its graphs by key (the pointers and sizes the launches bake
in), so a host that cycles through several input buffers replays as much as one that reuses one buffer, and a shape that
changes every tick runs only that stage directly.  Results must equal direct launches tick for tick.
Run on an H100:  python -m pytest tests -m gpu"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TICKS = 20
WARMUP = 12  # two cycles of the rotating build's 6 keys (3 position pairs x 2 key buffers)


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


def _run(chd, graphs, n_pos_buffers, batch_sizes=None):
    """TICKS ticks of TICK_ALL with device-resident positions: tick t reads position pair t mod n_pos_buffers, whose contents
    are rewritten before the tick.  batch_sizes: queries per tick (default: every subscriber).  -> (per-tick results,
    graph launches per tick)"""
    import torch

    wc = chd.synth.scaled(chd.synth.CONFIGS["benchmark"], 40_000, 4_000)
    e = chd.engine.Engine(wc.cfg(), wc.n_entities, wc.n_subscribers, max_visible=1 << 23)
    e.enable_graphs(graphs)
    ex, ez = chd.synth.entities(wc)
    conn, _, _, _ = chd.synth.subscribers(wc, ex, ez)
    e.set_subscribers(conn)
    pool = [(torch.empty(len(ex), dtype=torch.float64, device="cuda"), torch.empty(len(ex), dtype=torch.float64, device="cuda"))
            for _ in range(n_pos_buffers)]
    ring_state, res, launches = None, [], []
    for tick in range(TICKS):
        t = (tick + 1) * 33_000_000
        ex, ez = chd.synth.move_entities(wc, ex, ez, tick, 300.0)
        _, cx, cz, r = chd.synth.subscribers(wc, ex, ez)
        n = len(cx) if batch_sizes is None else batch_sizes[tick]
        ring_state, off, arr, snd, idx, cmi = chd.synth.update_rings(wc, tick, t, 33_000_000, 4, len(conn), ring_len=16, state=ring_state)
        e.set_rings(off, arr, snd, idx, cmi)
        tx, tz = pool[tick % n_pos_buffers]
        tx.copy_(torch.from_numpy(ex))
        tz.copy_(torch.from_numpy(ez))
        torch.cuda.synchronize()  # the last tick that read this pair has finished (its summary was read back)
        e.set_entities(tx, tz)
        batch, keep = chd.engine.make_batch(n, sub=np.arange(n, dtype=np.uint32), sphere=(cx[:n], cz[:n], r[:n]))
        g0 = e.graph_launch_count()
        s = e.tick(batch, t, chd.capi.TICK_ALL)
        launches.append(e.graph_launch_count() - g0)
        pairs = e.get_pairs(s.n_pairs)
        voff, vis = e.get_visible()
        due = e.get_due(s.n_due)
        due = due[np.lexsort((due["window_hi"], due["channel_id"], due["sub"]))]  # the due list is a set: canonical order
        res.append((s.as_dict(), pairs, voff, vis, due))
    e.close()
    return res, launches


def _assert_same(got, want):
    for tick, (a, b) in enumerate(zip(got, want)):
        assert a[0] == b[0], tick
        for k in b[1]:
            np.testing.assert_array_equal(a[1][k], b[1][k], err_msg=f"tick {tick} pairs {k}")
        for i, name in ((2, "vis_off"), (3, "vis"), (4, "due")):
            np.testing.assert_array_equal(a[i], b[i], err_msg=f"tick {tick} {name}")


def test_rotating_position_buffers_replay_like_one_buffer(chd):
    """Positions from a pool of three device buffer pairs: the build cycles through 6 keys and, after two cycles, replays
    on every tick as often as with one pair."""
    direct, none = _run(chd, False, 1)
    one, one_launches = _run(chd, True, 1)
    three, three_launches = _run(chd, True, 3)
    assert sum(none) == 0
    assert sum(r[0]["n_due"] for r in direct) > 1000
    _assert_same(one, direct)
    _assert_same(three, direct)
    assert min(one_launches[WARMUP:]) > 0
    assert three_launches[WARMUP:] == one_launches[WARMUP:]


def test_batch_size_changing_every_tick_runs_only_the_interest_update_direct(chd):
    """A query batch whose size changes every tick: the two interest-update graphs (the only keys holding the batch size)
    never replay, and every other stage replays as with a fixed batch size."""
    sizes = [4_000 - 1 - tick for tick in range(TICKS)]  # never the same twice
    direct, _ = _run(chd, False, 1, sizes)
    varying, varying_launches = _run(chd, True, 1, sizes)
    _, fixed_launches = _run(chd, True, 1)
    _assert_same(varying, direct)
    assert min(fixed_launches[WARMUP:]) > 2
    assert varying_launches[WARMUP:] == [n - 2 for n in fixed_launches[WARMUP:]]
