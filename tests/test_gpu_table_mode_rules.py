"""Mode rules of entity-table mode on slabs: an engine made a slab (chd_set_slab / chd_comm_init) before chd_entity_table_init
accepts the border export, the halo import and id-mode deltas; a table engine does not change its slab, and the calls that bypass
the table stay refused.  (tests/test_gpu_entity_table.py and tests/test_gpu_sharded_delta.py pin the refusals on a table engine
that is not a slab.)
Run on an H100:  python -m pytest tests/test_gpu_table_mode_rules.py -m gpu"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


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


def test_table_mode_on_a_slab_engine(chd):
    import torch

    cap = chd.capi
    L = cap.lib()
    wc = chd.synth.CONFIGS["2x2"]
    s = chd.engine.Engine(wc.cfg(), 64, 2)
    s.set_slab(0, 1, 1)
    s.entity_table_init()  # a slab may come first
    assert L.chd_set_slab(s.h, 0, 2, 1) == cap.ERR_STATE  # ... but not after
    uid = (C.c_uint8 * 128)()
    assert L.chd_comm_init(s.h, uid, 0, 1, 1, 16, 0, 0) == cap.ERR_STATE
    x, z, gid = np.zeros(4), np.zeros(4), np.arange(4, dtype=np.uint32)
    assert L.chd_set_entities(s.h, cap.ptr(x), cap.ptr(z), 4) == cap.ERR_STATE
    assert L.chd_set_entity_ids(s.h, cap.ptr(gid), 4) == cap.ERR_STATE
    assert L.chd_reserve_visible_delta(s.h, 64) == cap.ERR_STATE  # index mode stays single-GPU
    assert L.chd_reserve_visible_delta_ids(s.h, 64, 1 << 10) == cap.OK
    s.spawn_entities([5, 6], [-1000.0, 1000.0], [-1000.0, -1000.0])
    cnt = C.c_uint32()
    d = torch.full((32,), -1, dtype=torch.int32, device="cuda")
    # both are border records (column 0 borders the slab edge, column 1 lies beyond it), named by table id
    assert L.chd_export_border(s.h, cap.ptr(d), 16, C.byref(cnt)) == cap.OK and cnt.value == 2
    assert sorted(d[:4].cpu().numpy().view(np.uint32)[::2].tolist()) == [5, 6]
    assert L.chd_import_halo(s.h, cap.ptr(d), 2, 0, 2) == cap.OK
    s.build()
    assert sorted(s.get_cells()[1].tolist()) == [5, 6]
    # chd_entity_table_init stays refused after entity ids, a cell assignment, a build or id-mode deltas, slab or not
    for bad in ("ids", "assign", "build", "delta_ids"):
        f = chd.engine.Engine(wc.cfg(), 16, 2)
        f.set_slab(0, 1, 1)
        if bad == "ids":
            f.set_entity_ids(gid)
        elif bad == "assign":
            assert L.chd_assign_cells(f.h) == cap.OK
        elif bad == "build":
            f.set_entities(x, z)
            f.build()
        else:
            f.reserve_visible_delta_ids(64, 1 << 10)
        assert L.chd_entity_table_init(f.h) == cap.ERR_STATE, bad
        f.close()
    s.close()
