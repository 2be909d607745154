"""CPU-side checks of facings and follower frames (include/chd_gpu_facing.h): the header is plain C99 next to chd_gpu.h, the library
exports what it declares, every entry point refuses a NULL engine, the numpy restatement of the generation gives the answers derived
by hand, and the sharding helpers pass facings and frames through.  No GPU needed."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np

from tests._facing import frame_query

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "chd_gpu_facing.h")

def _declared():
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return sorted(set(re.findall(r"\b(chd_[a-z0-9_]+)\s*\(", src)))


def test_header_is_plain_c_and_frame_batch_matches(tmp_path):
    from channeld_b200 import capi

    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "chd_gpu.h"', '#include "chd_gpu_subs.h"', '#include "chd_gpu_facing.h"',
             'int main(void) {', '  printf("size %zu\\n", sizeof(chd_follow_frame_batch));']
    for fname, _ in capi.FollowFrameBatch._fields_:
        lines.append('  printf("%s %%zu\\n", offsetof(chd_follow_frame_batch, %s));' % (fname, fname))
    lines += ['  return 0;', '}']
    src = tmp_path / "facing_layout.c"
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "facing_layout"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = dict(l.split(" ", 1) for l in subprocess.check_output([str(exe)], text=True).splitlines())
    assert int(got["size"]) == C.sizeof(capi.FollowFrameBatch)
    for fname, _ in capi.FollowFrameBatch._fields_:
        assert int(got[fname]) == getattr(capi.FollowFrameBatch, fname).offset, fname


def test_library_exports_every_declared_symbol():
    from channeld_b200 import capi

    L = capi.lib()
    names = _declared()
    for n in names:
        assert hasattr(L, n), "libchd_b200.so does not export %s" % n
    assert sorted(capi.FACING_SYMBOLS) == names
    assert not set(capi.FACING_SYMBOLS) & (set(capi.SYMBOLS) | set(capi.SUB_SYMBOLS))


def test_null_engine_is_an_error_everywhere():
    code = '''
import ctypes as C, sys
sys.path.insert(0, %r)
from channeld_b200 import capi
L = capi.lib()
bad = []
for name in capi.FACING_SYMBOLS:
    f = getattr(L, name)
    assert f.argtypes is not None, name
    args = [0.0 if t is C.c_double else (None if (t is C.c_void_p or hasattr(t, "contents")) else 0) for t in f.argtypes]
    if f(*args) != capi.ERR_INVALID:
        bad.append(name)
b = capi.FollowFrameBatch(n=0)
if L.chd_follow_set_frame(None, C.byref(b)) != capi.ERR_INVALID:
    bad.append("chd_follow_set_frame(NULL, batch)")
n = C.c_uint32()
if L.chd_handoff_entities_facing(None, None, None, None, None, None, None, 0, C.byref(n)) != capi.ERR_INVALID:
    bad.append("chd_handoff_entities_facing(NULL, count)")
print("BAD", bad)
''' % ROOT
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "BAD []" in out.stdout, out.stdout


# ---- the numpy restatement against answers derived by hand

def _q(fx, fz, fwd=0.0, right=0.0, rot=(1.0, 0.0), x=500.0, z=700.0, cone=(0.6, 0.8)):
    return [float(v) for v in frame_query(x, z, fx, fz, fwd, right, rot[0], rot[1], cone[0], cone[1])]


def test_forward_offset_moves_the_centre_along_the_facing():
    fx, fz, cx, cz, dx, dz = _q(0.0, 1.0, fwd=100.0)
    assert (cx, cz) == (500.0, 800.0) and (dx, dz) == (0.0, 1.0) and (fx, fz) == (0.0, 1.0)
    assert _q(1.0, 0.0, fwd=100.0)[2:4] == [600.0, 700.0]
    assert _q(0.0, 2.0, fwd=100.0)[2:4] == [500.0, 800.0]  # the offset takes the unit facing


def test_right_offset_is_the_pawns_right():
    # facing +z: the right-hand side (-uz, ux) is -x
    assert _q(0.0, 1.0, right=50.0)[2:4] == [450.0, 700.0]
    # facing +x: the right-hand side is +z (UE's +Y after the Y <-> Z swap)
    assert _q(1.0, 0.0, right=50.0)[2:4] == [500.0, 750.0]


def test_cone_rotation():
    assert _q(1.0, 0.0, rot=(0.0, 1.0))[4:6] == [0.0, 1.0]  # 90 degrees maps (1, 0) to (0, 1)
    assert _q(0.0, 1.0, rot=(0.0, 1.0))[4:6] == [-1.0, 0.0]
    assert _q(0.3, -0.4)[4:6] == [0.3, -0.4]  # the identity keeps the facing exactly


def test_no_facing_gives_the_plain_query():
    plain = [0.0, 0.0, 500.0, 700.0, 0.6, 0.8]
    for fx, fz in ((0.0, 0.0), (-0.0, 0.0), (np.nan, 1.0), (1.0, np.inf), (-np.inf, 0.0)):
        assert _q(fx, fz, fwd=100.0, right=50.0, rot=(0.0, 1.0)) == plain, (fx, fz)


def test_router_and_registry_pass_facings_and_frames_through():
    from channeld_b200.sharding import EntityRouter, FollowerRegistry

    r = EntityRouter(2, 8, 0.0, 100.0)
    ids = np.array([1, 2, 3], np.uint32)
    x, z = np.array([50.0, 650.0, 150.0]), np.array([1.0, 2.0, 3.0])
    fx, fz = np.array([1.0, 0.0, 0.6]), np.array([0.0, 1.0, 0.8])
    plain = r.spawn(ids, x, z)
    assert [len(b) for b in plain] == [3, 3]
    r2 = EntityRouter(2, 8, 0.0, 100.0)
    sp = r2.spawn(ids, x, z, fx, fz)
    assert [b[0].tolist() for b in sp] == [[1, 3], [2]]
    np.testing.assert_array_equal(sp[0][3], [1.0, 0.6])
    np.testing.assert_array_equal(sp[1][4], [1.0])
    mv = r2.move(ids, x, z, fx, fz)
    assert [len(b) for b in mv] == [5, 5] and mv[0][4].tolist() == [0.0, 0.8]
    assert [len(b) for b in r2.move(ids, x, z)] == [3, 3]
    # hand-off lists with facings become facing spawns at the destination
    lists = [(np.array([3], np.uint32), np.array([1], np.uint32), np.array([420.0]), np.array([3.0]), np.array([0.6]), np.array([0.8])),
             (np.zeros(0, np.uint32), np.zeros(0, np.uint32), np.zeros(0), np.zeros(0), np.zeros(0), np.zeros(0))]
    ad = r2.handoff(lists)
    assert r2.owner[3] == 1 and [len(b) for b in ad] == [5, 5]
    assert ad[1][0].tolist() == [3] and ad[1][1].tolist() == [420.0] and ad[1][3].tolist() == [0.6] and ad[1][4].tolist() == [0.8]
    assert [len(b) for b in r2.handoff([l[:4] for l in lists])] == [3, 3]
    # a plain list beside a facing one: its entities get no facing, every column keeps one entry per id
    mixed = EntityRouter(2, 8, 0.0, 100.0).handoff([(np.array([1], np.uint32), np.array([1], np.uint32), np.array([700.0]), np.array([1.0])), lists[0]])
    assert mixed[1][0].tolist() == [1, 3] and mixed[1][3].tolist() == [0.0, 0.6] and mixed[1][4].tolist() == [0.0, 0.8]
    assert all(len(c) == 2 for c in mixed[1])
    # the registry: frames ride with the bind batches of their connections
    reg = FollowerRegistry(2)
    shape = (50.0, 0, 0, 1.0, 0.0, 0.5, 80.0)
    reg.follow(10, 1, 8, shape, frame=(100.0, -20.0))
    reg.follow(11, 2, 8, shape)
    reg.follow(12, 3, 8, shape, frame=(0.0, 0.0, 0.0, 1.0))
    binds = reg.plan(r2)[4]
    assert binds[0]["conn"] == [10] and binds[1]["conn"] == [11, 12]
    f0, f1 = binds[0]["frame"], binds[1]["frame"]
    assert f0["slot"].tolist() == binds[0]["slot"].tolist() and f0["off_fwd"].tolist() == [100.0] and f0["off_right"].tolist() == [-20.0]
    assert f0["rot_cos"].tolist() == [1.0] and f0["rot_sin"].tolist() == [0.0]
    assert f1["slot"].tolist() == [binds[1]["slot"][1]] and f1["rot_sin"].tolist() == [1.0]
    # re-following without a frame makes the follower plain; a batch without framed followers has no frame entry
    reg.follow(12, 3, 8, shape)
    b = reg.plan(r2)[4]
    assert b[1]["conn"] == [12] and "frame" not in b[1]
