"""CPU-side checks of the drop-in boundary: the C-ABI library builds for sm_90a, loads, and exports every
symbol include/chd_gpu.h declares.  No compute calls: these run without a GPU."""
import ctypes as C
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "chd_gpu.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(chd_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from channeld_b200 import capi

    L = capi.lib()
    names = _declared()
    assert len(names) >= 35
    for n in names:
        assert hasattr(L, n), "libchd_b200.so does not export %s" % n
    assert sorted(capi.SYMBOLS) == names
    assert L.chd_abi_version() == 1


def test_struct_layouts_match_header():
    from channeld_b200 import capi

    assert C.sizeof(capi.GridCfg) == 4 * 8 + 6 * 4
    assert C.sizeof(capi.Limits) == 4 * 4 + 3 * 8 + 4 * 4
    assert C.sizeof(capi.Due) == 48
    assert C.sizeof(capi.TickSummary) == 2 * 8 + 8 * 4 + 3 * 8 + 2 * 4
    assert C.sizeof(capi.QueryBatch) == 8 + 20 * 8


def test_header_is_plain_c_and_ctypes_mirrors_it(tmp_path):
    """include/chd_gpu.h compiles as C99 (it is what cgo / JNI / ctypes bind) and every struct the Python binding
    mirrors has the size and field offsets the C compiler gives it."""
    import subprocess

    from channeld_b200 import capi

    pairs = [("chd_grid_cfg", capi.GridCfg), ("chd_limits", capi.Limits), ("chd_query_batch", capi.QueryBatch), ("chd_due", capi.Due),
             ("chd_tick_summary", capi.TickSummary), ("chd_result_buffers", capi.ResultBuffers), ("chd_broadcast_batch", capi.BroadcastBatch)]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "chd_gpu.h"', 'int main(void) {']
    for cname, cls in pairs:
        lines.append('  printf("%s %%zu\\n", sizeof(%s));' % (cname, cname))
        for fname, _ in cls._fields_:
            lines.append('  printf("%s.%s %%zu\\n", offsetof(%s, %s));' % (cname, fname, cname, fname))
    lines += ['  return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())
    for cname, cls in pairs:
        assert int(got[cname]) == C.sizeof(cls), cname
        for fname, _ in cls._fields_:
            assert int(got["%s.%s" % (cname, fname)]) == getattr(cls, fname).offset, (cname, fname)


def test_c_example_compiles_links_and_fails_loudly_without_gpu(tmp_path):
    """examples/tick_loop.c (the pipelined host loop in plain C99) builds against the header and the library; on a box
    without a GPU it stops at chd_create with the 'no CPU fallback' error instead of computing anything."""
    import subprocess

    from channeld_b200 import capi

    lib_dir = os.path.dirname(capi.lib_path())
    exe = tmp_path / "tick_loop"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "examples", "tick_loop.c"), "-L", lib_dir, "-lchd_b200", "-Wl,-rpath," + lib_dir,
                           "-Wl,-rpath,/usr/local/cuda/lib64", "-L/usr/local/cuda/lib64", "-o", str(exe)])
    import torch

    if not torch.cuda.is_available():
        out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
        assert out.returncode == 2 and "no CPU fallback" in out.stderr


def test_null_engine_is_an_error_everywhere():
    """Error behaviour of the boundary: every entry point that takes an engine handle returns CHD_ERR_INVALID for a NULL
    handle (no crash, no CUDA call).  Runs in a subprocess so that a missing check cannot take pytest down with it."""
    import subprocess
    import sys

    code = '''
import ctypes as C, sys
sys.path.insert(0, %r)
from channeld_b200 import capi
L = capi.lib()
no_handle = {"chd_abi_version", "chd_default_limits", "chd_create", "chd_destroy", "chd_last_error", "chd_alloc_pinned", "chd_free_pinned", "chd_device_numa_node",
             "chd_get_adjacent_channels", "chd_get_regions", "chd_damping_interval_ms", "chd_launch_count", "chd_graph_launch_count",
             "chd_collective_count", "chd_comm_exchange_mode"}
bad = []
for name in capi.SYMBOLS:
    if name in no_handle:
        continue
    f = getattr(L, name)
    assert f.argtypes is not None, name
    args = [0.0 if t is C.c_double else (None if (t is C.c_void_p or hasattr(t, "contents")) else 0) for t in f.argtypes]
    if f(*args) != capi.ERR_INVALID:
        bad.append(name)
L.chd_destroy(None)
assert L.chd_launch_count(None) == 0 and L.chd_graph_launch_count(None) == 0 and L.chd_collective_count(None) == 0
print("BAD", bad)
''' % ROOT
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "BAD []" in out.stdout, out.stdout


def test_host_helpers_match_oracle(oracle):
    """GetAdjacentChannels / GetRegions / damping are plain host integer math in the library: checked here."""
    from channeld_b200 import capi
    from channeld_b200.engine import grid_cfg
    from tests._oracle import make_grid

    L = capi.lib()
    for g in [(0, 0, 10, 10, 1, 1, 1, 1), (-5, -5, 5, 5, 2, 2, 1, 1), (-40, -60, 20, 40, 4, 3, 2, 3), (-15000, -15000, 2000, 2000, 15, 15, 3, 3)]:
        cfg = grid_cfg(*g)
        og = make_grid(*g)
        n = g[4] * g[5]
        for cid in range(65536, 65536 + n):
            out = np.zeros(8, np.uint32)
            k = L.chd_get_adjacent_channels(C.byref(cfg), cid, capi.ptr(out))
            assert [int(v) for v in out[:k]] == oracle.adjacent(og, cid)
        a = [np.zeros(n) for _ in range(4)]
        cid, srv = np.zeros(n, np.uint32), np.zeros(n, np.uint32)
        assert L.chd_get_regions(C.byref(cfg), *[capi.ptr(v) for v in a], capi.ptr(cid), capi.ptr(srv)) == 0
        want = oracle.regions(og)
        for got, w in zip(a + [cid, srv], want):
            np.testing.assert_array_equal(got, w)
    for d in range(6):
        assert L.chd_damping_interval_ms(d, 33) == oracle.damping(d, 33)


def test_create_without_gpu_fails_loudly():
    import torch

    if torch.cuda.is_available():
        return
    from channeld_b200 import capi
    from channeld_b200.engine import Engine, grid_cfg

    try:
        Engine(grid_cfg(0, 0, 10, 10, 1, 1), 16, 16)
    except capi.ChdError as e:
        assert e.status == capi.ERR_CUDA and "no CPU fallback" in str(e)
    else:
        raise AssertionError("engine creation must fail without a CUDA device")


def test_create_validates_like_load_config():
    from channeld_b200 import capi
    from channeld_b200.engine import grid_cfg

    L = capi.lib()
    h = C.c_void_p()
    for bad in [grid_cfg(0, 0, 0, 10, 1, 1), grid_cfg(0, 0, 10, -1, 1, 1), grid_cfg(0, 0, 10, 10, 0, 1), grid_cfg(0, 0, 10, 10, 1, 1, 0, 1)]:
        assert L.chd_create(C.byref(bad), None, 0, C.byref(h)) == capi.ERR_INVALID
        assert b"should be positive" in L.chd_last_error(None)


def test_cpp_host_mirror_compiles(tmp_path):
    """channeld_b200/host/spatial_controller.hpp (the C++ mirror of the SpatialController interface) compiles
    against include/chd_gpu.h and links with the library."""
    import subprocess

    from channeld_b200 import capi

    src = tmp_path / "host_check.cpp"
    src.write_text('#include "channeld_b200/host/spatial_controller.hpp"\n'
                   '// instantiate the whole method set (never called: there is no GPU on the build host)\n'
                   'void use_all(channeld::GpuStaticGrid2DSpatialController& c, const chd_query_batch& b, const chd_result_buffers& rb) {\n'
                   '  chd_tick_summary s{}; c.PrefetchEntities(nullptr, nullptr, 0); c.PrefetchQueries(b);\n'
                   '  c.PrefetchRings(nullptr, 0, nullptr, nullptr, nullptr, nullptr); c.AdoptPrefetched(); c.BeginInterest(nullptr, 0);\n'
                   '  c.Tick(nullptr, 0, CHD_TICK_ALL | CHD_TICK_EARLY_RESULTS); c.FetchResults(rb, &s);\n'
                   '  c.AdjacentBroadcast({65536}, {64}, {}, {}, 16); c.GetDueClasses(s.n_due); }\n'
                   'int main() { channeld::GpuStaticGrid2DSpatialController c; return c.GetAdjacentChannels(65536).size() == 0 ? 0 : 1; }\n')
    lib_dir = os.path.dirname(capi.lib_path())
    exe = tmp_path / "host_check"
    subprocess.check_call(["g++", "-std=c++17", "-I", ROOT, str(src), "-L", lib_dir, "-lchd_b200", "-Wl,-rpath," + lib_dir,
                           "-Wl,-rpath,/usr/local/cuda/lib64", "-L/usr/local/cuda/lib64", "-o", str(exe)])
