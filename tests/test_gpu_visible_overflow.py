"""CHD_OVF_VISIBLE far above capacity: a tick whose expanded visible list needs many times chd_limits.max_visible entries reports the
overflow and the entries it needed, writes nothing past its buffers, and the next tick within capacity gives the oracle's lists.
The engine takes the CTA-tile emit path here (at least EMIT_TILE / 2 entities per cell), whose tile descriptors hold one entry per
2048 entries of max_visible: the partition must stop at that count, not at the twice larger count of 1024-entry warp tiles.
Run on an H100:  python -m pytest tests/test_gpu_visible_overflow.py -m gpu"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

GRID = (-200.0, -200.0, 100.0, 100.0, 4, 4)  # 16 cells


@pytest.mark.parametrize("graphs", [True, False], ids=["graphs", "direct"])
def test_visible_overflow_far_above_capacity(oracle, graphs):
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from channeld_b200 import capi, engine
    from tests._oracle import make_grid

    rng = np.random.default_rng(11)
    N, S, cap = 40_000, 80, 1 << 20  # 2 500 entities per cell
    ex, ez = -200 + rng.random(N) * 400, -200 + rng.random(N) * 400
    e = engine.Engine(engine.grid_cfg(*GRID), N, S, max_visible=cap)
    e.enable_graphs(graphs)
    e.set_entities(ex, ez)
    e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
    sub = np.arange(S, dtype=np.uint32)
    g = make_grid(*GRID)
    for k, big in enumerate((True, True, False, False, True, False)):
        cx, cz = -150 + rng.random(S) * 300, -150 + rng.random(S) * 300
        r = np.full(S, 800.0 if big else 20.0)  # every cell (V = S x N = 3.2 M entries, 3 x max_visible) or one to four cells
        batch, keep = engine.make_batch(S, sub=sub, sphere=(cx, cz, r))
        s = e.tick(batch, (k + 1) * 33_000_000, capi.TICK_BUILD | capi.TICK_EMIT, want_summary=False)
        st = capi.TickSummary()
        rc = e.L.chd_summary(e.h, C.byref(st))
        want = oracle.sphere_tick(g, ex, ez, cx, cz, r)
        V = int(want["vis_off"][-1])
        assert st.n_visible == st.required_visible == V
        if big:
            assert V > 2 * cap and rc == capi.ERR_CAPACITY and st.overflow == capi.OVF_VISIBLE
            continue
        assert V <= cap and rc == capi.OK and st.overflow == 0
        voff, vis = e.get_visible()
        np.testing.assert_array_equal(voff, want["vis_off"])
        np.testing.assert_array_equal(vis, want["vis_entity"])
    e.close()
