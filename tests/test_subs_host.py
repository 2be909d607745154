"""CPU-side checks of explicit subscriptions (include/chd_gpu_subs.h): the header is plain C99 next to chd_gpu.h, the library exports
what it declares, every entry point refuses a NULL engine, and the oracle's presence-mask merge gives the answers derived by hand
from subscription.go:34-125.  No GPU needed."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from tests._subs_oracle import (ERR_CHANNEL, ERR_SLOT, MERGED, NEW, NOT_SUBSCRIBED, OPT_DELAY, OPT_INTERVAL, OPT_SKIP_FIRST, OPT_SKIP_SELF,
                                SUB, UNSUB, UNSUBSCRIBED, DIST_EXPLICIT, SubsOracle)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "chd_gpu_subs.h")

def _declared():
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return sorted(set(re.findall(r"\b(chd_[a-z0-9_]+)\s*\(", src)))


def test_header_is_plain_c_and_sub_batch_matches(tmp_path):
    from channeld_b200 import capi

    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "chd_gpu.h"', '#include "chd_gpu_subs.h"', 'int main(void) {',
             '  printf("size %zu\\n", sizeof(chd_sub_batch));']
    for fname, _ in capi.SubBatch._fields_:
        lines.append('  printf("%s %%zu\\n", offsetof(chd_sub_batch, %s));' % (fname, fname))
    lines.append('  printf("consts %d %d %d %d %u\\n", CHD_SUBOP_UNSUB, CHD_SUBOPT_SKIP_FIRST, CHD_SUB_NOT_SUBSCRIBED, CHD_SUB_ERR_CAPACITY, '
                 'CHD_DIST_EXPLICIT);')
    lines += ['  return 0;', '}']
    src = tmp_path / "subs_layout.c"
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "subs_layout"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = subprocess.check_output([str(exe)], text=True).splitlines()
    got = dict(l.split(" ", 1) for l in out)
    assert int(got["size"]) == C.sizeof(capi.SubBatch)
    for fname, _ in capi.SubBatch._fields_:
        assert int(got[fname]) == getattr(capi.SubBatch, fname).offset, fname
    assert got["consts"].split() == [str(v) for v in (capi.SUBOP_UNSUB, capi.SUBOPT_SKIP_FIRST, capi.SUB_NOT_SUBSCRIBED, capi.SUB_ERR_CAPACITY,
                                                      capi.DIST_EXPLICIT)]


def test_library_exports_every_declared_symbol():
    from channeld_b200 import capi

    L = capi.lib()
    names = _declared()
    for n in names:
        assert hasattr(L, n), "libchd_b200.so does not export %s" % n
    assert sorted(capi.SUB_SYMBOLS) == names
    assert not set(capi.SUB_SYMBOLS) & set(capi.SYMBOLS)


def test_null_engine_is_an_error_everywhere():
    code = '''
import ctypes as C, sys
sys.path.insert(0, %r)
from channeld_b200 import capi
L = capi.lib()
bad = []
for name in capi.SUB_SYMBOLS:
    f = getattr(L, name)
    assert f.argtypes is not None, name
    args = [0.0 if t is C.c_double else (None if (t is C.c_void_p or hasattr(t, "contents")) else 0) for t in f.argtypes]
    if f(*args) != capi.ERR_INVALID:
        bad.append(name)
b = capi.SubBatch(n=0)
if L.chd_apply_subscriptions(None, C.byref(b), 0, None) != capi.ERR_INVALID:
    bad.append("chd_apply_subscriptions(NULL, batch)")
print("BAD", bad)
''' % ROOT
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "BAD []" in out.stdout, out.stdout


# ---- the oracle's merge, against answers derived by hand from subscription.go:34-125 (conn 7 on slot 0, channel 0x10000 = cell 0)

@pytest.fixture
def orc():
    from tests import _oracle

    return _oracle.load()


def _one(o, op, now, present=0, interval=0, delay=0, skip_self=0, skip_first=0, slot=0, channel=0x10000):
    return int(o.apply([slot], [channel], [op], now, present=np.array([present], np.uint8), interval=[interval], delay=[delay],
                       skip_self=[skip_self], skip_first=[skip_first])[0])


def test_oracle_defaults(orc):
    o = SubsOracle(orc, 4, [7], default_interval_ms=50, default_delay_ms=3)
    assert _one(o, SUB, 1_000_000_000) == NEW
    t = o.table(1)
    assert list(t["interval"]) == [50] and list(t["dist"]) == [DIST_EXPLICIT] and list(t["skip_self"]) == [True]
    last, had, li = o.state()
    assert last[0] == 1_000_000_000 + 3_000_000 and not had[0] and li[0] == 0  # lastFanOutTime = now + FanOutDelayMs


def test_oracle_delay_and_skip_first_at_creation_only(orc):
    o = SubsOracle(orc, 4, [7], default_interval_ms=50)
    assert _one(o, SUB, 1_000_000_000, OPT_DELAY | OPT_SKIP_FIRST, delay=40, skip_first=1) == NEW
    last, had, _ = o.state()
    assert last[0] == 1_040_000_000 and had[0]
    assert _one(o, SUB, 2_000_000_000, OPT_DELAY | OPT_SKIP_FIRST, delay=900, skip_first=0) == MERGED
    last2, had2, _ = o.state()
    assert last2[0] == 1_040_000_000 and had2[0]  # unchanged


def test_oracle_skip_self_and_interval_merged(orc):
    o = SubsOracle(orc, 4, [7], default_interval_ms=50)
    assert _one(o, SUB, 0, OPT_INTERVAL | OPT_SKIP_SELF, interval=100, skip_self=0) == NEW
    t = o.table(1)
    assert list(t["interval"]) == [100] and list(t["skip_self"]) == [False]
    assert _one(o, SUB, 5, OPT_SKIP_SELF, skip_self=1) == MERGED  # only SkipSelf present: the interval stays
    t = o.table(1)
    assert list(t["interval"]) == [100] and list(t["skip_self"]) == [True]
    assert _one(o, SUB, 6, OPT_INTERVAL, interval=30) == MERGED  # only the interval present: SkipSelf stays
    t = o.table(1)
    assert list(t["interval"]) == [30] and list(t["skip_self"]) == [True]
    assert _one(o, SUB, 7) == MERGED  # nothing present: nothing changes
    assert list(o.table(1)["interval"]) == [30]


def test_oracle_max_interval_raised_at_creation_only(orc):
    o = SubsOracle(orc, 4, [7, 8], default_interval_ms=50)
    assert _one(o, SUB, 0, OPT_INTERVAL, interval=80) == NEW
    assert _one(o, SUB, 0, OPT_INTERVAL, interval=500) == MERGED
    assert list(o.ch.get_rings()["max_interval_ms"]) == [80, 0, 0, 0]
    assert _one(o, SUB, 0, OPT_INTERVAL, interval=200, slot=1) == NEW
    assert list(o.ch.get_rings()["max_interval_ms"]) == [200, 0, 0, 0]


def test_oracle_statuses_in_array_order(orc):
    o = SubsOracle(orc, 4, [7, 0], default_interval_ms=50)
    st = o.apply([0, 0, 0, 0, 1, 0, 2], [0x10001, 0x10001, 0x10001, 0x10001, 0x10001, 0x10004, 0x10000], [SUB, SUB, UNSUB, UNSUB, SUB, SUB, SUB], 0)
    assert list(st) == [NEW, MERGED, UNSUBSCRIBED, NOT_SUBSCRIBED, ERR_SLOT, ERR_CHANNEL, ERR_SLOT]
    assert o.pairs == {}
