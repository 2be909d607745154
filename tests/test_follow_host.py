"""Host layers of the followers (no GPU): the ctypes prototypes of the chd_follow_* entry points and the controller's translation of
SpatialInterestQuery shapes into a binding batch."""
import ctypes as C

import numpy as np
import pytest


def test_capi_declares_the_follow_entry_points():
    from channeld_b200 import capi

    L = capi.lib()
    want = {"chd_follow_bind": 2, "chd_follow_unbind": 3, "chd_follow_queries": 2, "chd_get_follow": 9}
    for name, nargs in want.items():
        assert name in capi.SYMBOLS
        f = getattr(L, name)
        assert f.restype is C.c_int and len(f.argtypes) == nargs, name
    assert C.sizeof(capi.FollowBatch) == 8 + 10 * 8
    assert (capi.FOLLOW_ALL, capi.FOLLOW_MOVED, capi.FOLLOW_NOT_SELECTED, capi.FOLLOW_NO_ENTITY, capi.TICK_FOLLOW) == (0, 1, 16, 17, 32)
    assert capi.STAGE_FOLLOW == 12


def test_follow_batch_layout_matches_header(tmp_path):
    import os
    import subprocess

    from channeld_b200 import capi

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "chd_gpu.h"', 'int main(void) {', '  printf("size %zu\\n", sizeof(chd_follow_batch));']
    lines += ['  printf("%s %%zu\\n", offsetof(chd_follow_batch, %s));' % (f, f) for f, _ in capi.FollowBatch._fields_]
    lines += ['  return CHD_FOLLOW_ALL + CHD_FOLLOW_MOVED + CHD_FOLLOW_NOT_SELECTED + CHD_FOLLOW_NO_ENTITY + CHD_TICK_FOLLOW + CHD_STAGE_FOLLOW - 78;', '}']
    src = tmp_path / "follow.c"
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "follow"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)])
    got = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())
    assert int(got["size"]) == C.sizeof(capi.FollowBatch)
    for f, _ in capi.FollowBatch._fields_:
        assert int(got[f]) == getattr(capi.FollowBatch, f).offset, f


class StubEngine:
    def __init__(self):
        self.calls = []

    def follow_bind(self, slots, entities, **kw):
        self.calls.append(("bind", list(slots), list(entities), kw))

    def follow_unbind(self, slots):
        self.calls.append(("unbind", list(slots)))

    def follow_queries(self, mode):
        self.calls.append(("queries", mode))

    def tick(self, batch, t_ns, flags):
        self.calls.append(("tick", batch, t_ns, flags))
        return "summary"


def test_controller_translates_shapes_and_ignores_centres():
    from channeld_b200 import capi
    from channeld_b200 import controller as c

    ctl = c.GpuStaticGrid2DSpatialController()
    ctl.engine = StubEngine()
    far = c.SpatialInfo(1e9, 0, -1e9)  # centres are ignored: the followed entity is the centre
    qs = [c.SpatialInterestQuery(SphereAOI=c.SphereAOI(far, 50.0)),
          c.SpatialInterestQuery(BoxAOI=c.BoxAOI(far, c.SpatialInfo(10, 99, 20))),
          c.SpatialInterestQuery(ConeAOI=c.ConeAOI(None, c.SpatialInfo(0.6, 0, 0.8), 0.5, 70.0), SphereAOI=c.SphereAOI(None, 5.0))]
    ctl.FollowEntities([3, 4, 9], [100, 200, 300], qs)
    (op, slots, ents, kw), = ctl.engine.calls
    assert (op, slots, ents) == ("bind", [3, 4, 9], [100, 200, 300])
    assert kw["kind"].tolist() == [capi.AOI_SPHERE, capi.AOI_BOX, capi.AOI_CONE | capi.AOI_SPHERE]
    assert kw["sph_r"].tolist() == [50.0, 0.0, 5.0]
    assert [a.tolist() for a in kw["box"]] == [[0, 10, 0], [0, 20, 0]]
    assert [a.tolist() for a in kw["cone"]] == [[0, 0, 0.6], [0, 0, 0.8], [0, 0, 0.5], [0, 0, 70.0]]
    with pytest.raises(c.SpatialError):
        ctl.FollowEntities([1], [1], [c.SpatialInterestQuery(SpotsAOI=c.SpotsAOI([far], []))])
    with pytest.raises(c.SpatialError):
        ctl.FollowEntities([1], [1], [c.SpatialInterestQuery()])
    with pytest.raises(c.SpatialError):
        ctl.FollowEntities([1], [1], [c.SpatialInterestQuery(BoxAOI=c.BoxAOI(far, None))])
    assert len(ctl.engine.calls) == 1
    ctl.UnfollowEntities([4])
    assert ctl.Tick(None, 33, follow=capi.FOLLOW_MOVED) == "summary"
    assert ctl.engine.calls[1:] == [("unbind", [4]), ("queries", capi.FOLLOW_MOVED), ("tick", None, 33, capi.TICK_ALL | capi.TICK_FOLLOW)]
    with pytest.raises(c.SpatialError):
        ctl.Tick(object(), 33, follow=capi.FOLLOW_ALL)
