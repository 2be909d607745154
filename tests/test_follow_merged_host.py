"""Host layers of merged interest updates (chd_follow_queries_with), without a GPU: the ctypes prototype, the header's new enumerator
and prototype, the host part's size class and the controller's explicit= translation."""
import ctypes as C
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_capi_declares_follow_queries_with():
    from channeld_b200 import capi

    L = capi.lib()
    assert "chd_follow_queries_with" in capi.SYMBOLS
    f = L.chd_follow_queries_with
    assert f.restype is C.c_int and len(f.argtypes) == 3
    assert f.argtypes[1] is C.c_uint32 and f.argtypes[2]._type_ is capi.QueryBatch
    assert capi.FOLLOW_OVERRIDDEN == 18


def test_header_declares_the_overridden_status_and_the_prototype(tmp_path):
    src = tmp_path / "merged.c"
    src.write_text('#include "chd_gpu.h"\n'
                   'static chd_status (*const fn)(chd_engine*, uint32_t, const chd_query_batch*) = chd_follow_queries_with;\n'
                   'int main(void) { return (fn != 0) + CHD_FOLLOW_OVERRIDDEN - CHD_FOLLOW_NO_ENTITY - 2; }\n')
    exe = tmp_path / "merged"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-c", "-I", os.path.join(ROOT, "include"), str(src), "-o",
                           str(exe) + ".o"])
    obj = tmp_path / "value.c"  # the enumerator's value, compiled and run
    obj.write_text('#include <stdio.h>\n#include "chd_gpu.h"\nint main(void) { printf("%d\\n", (int)CHD_FOLLOW_OVERRIDDEN); return 0; }\n')
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(obj), "-o", str(exe)])
    assert subprocess.check_output([str(exe)], text=True).strip() == "18"


@pytest.mark.parametrize("n, H", [(0, 0), (1, 256), (255, 256), (256, 256), (257, 512), (512, 512), (513, 1024), ((1 << 17) + 1, 1 << 18),
                                  (1 << 20, 1 << 20)])
def test_host_part_size(n, H):
    from channeld_b200.engine import host_part_size

    assert host_part_size(n) == H


class StubEngine:
    def __init__(self):
        self.calls = []

    def follow_queries(self, mode):
        self.calls.append(("queries", mode))

    def follow_queries_with(self, mode, batch=None):
        self.calls.append(("queries_with", mode, batch))

    def tick(self, batch, t_ns, flags):
        self.calls.append(("tick", batch, t_ns, flags))
        return "summary"


def test_controller_merges_explicit_queries_into_a_followed_tick():
    from channeld_b200 import capi
    from channeld_b200 import controller as c

    ctl = c.GpuStaticGrid2DSpatialController()
    ctl.engine = StubEngine()
    explicit = object()
    assert ctl.Tick(None, 33, follow=capi.FOLLOW_MOVED, explicit=explicit) == "summary"
    assert ctl.Tick(None, 66, capi.TICK_BUILD, follow=capi.FOLLOW_ALL) == "summary"
    assert ctl.engine.calls == [("queries_with", capi.FOLLOW_MOVED, explicit), ("tick", None, 33, capi.TICK_ALL | capi.TICK_FOLLOW),
                                ("queries", capi.FOLLOW_ALL), ("tick", None, 66, capi.TICK_BUILD | capi.TICK_FOLLOW)]
    with pytest.raises(c.SpatialError):
        ctl.Tick(object(), 99, follow=capi.FOLLOW_ALL, explicit=explicit)
    with pytest.raises(c.SpatialError):
        ctl.Tick(None, 99, explicit=explicit)
    assert len(ctl.engine.calls) == 4
