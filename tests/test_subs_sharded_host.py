"""CPU-side checks of explicit subscriptions on slabs (include/chd_gpu_subs_sharded.h): the header is plain C99 after chd_gpu.h, the
library exports what it declares, a NULL engine is refused, the entry point declares the needs and applies the call-order rules of
chd_apply_subscriptions plus rule 12's staged updates, and sharding.route_sub_ops / merge_sub_status split and join a batch named by
subscriber keys.  No GPU needed."""
import os
import re
import subprocess
import sys

import numpy as np

from tests.test_entry_points import ALWAYS, NEEDS, _bodies, _chain_variants, _flags

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "chd_gpu_subs_sharded.h")
ENTRY = "chd_apply_subscriptions_sharded"


def _uncommented(path=HEADER):
    return re.sub(r"/\*.*?\*/", "", open(path).read(), flags=re.S)


def _declared():
    return sorted(set(re.findall(r"\b(chd_[a-z0-9_]+)\s*\(", _uncommented())))


def test_header_is_plain_c_and_its_status_is_distinct(tmp_path):
    from channeld_b200 import capi

    src = tmp_path / "subs_sharded_hdr.c"
    src.write_text('#include "chd_gpu.h"\n#include "chd_gpu_subs_sharded.h"\n#include "chd_gpu_subs_sharded.h"\n#include <stdio.h>\n'
                   "int main(void) { chd_status (*f)(chd_engine*, const chd_sub_batch*, int64_t, uint8_t*) = chd_apply_subscriptions_sharded;\n"
                   '  printf("%d\\n", (int)CHD_SUB_ERR_OUTSIDE_SLAB); return f == 0; }\n')
    obj = tmp_path / "subs_sharded_hdr.o"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src), "-c", "-o", str(obj)])
    value = int(re.search(r"CHD_SUB_ERR_OUTSIDE_SLAB\s*=\s*(\d+)", _uncommented()).group(1))
    assert value == capi.SUB_ERR_OUTSIDE_SLAB
    subs = {int(v) for v in re.findall(r"\bCHD_SUB_[A-Z_]+\s*=\s*(\d+)", _uncommented(os.path.join(ROOT, "include", "chd_gpu_subs.h")))}
    assert len(subs) == 7 and value not in subs


def test_library_exports_every_declared_symbol():
    from channeld_b200 import capi

    L = capi.lib()
    names = _declared()
    for n in names:
        assert hasattr(L, n), "libchd_b200.so does not export %s" % n
    assert sorted(capi.SUB_SHARDED_SYMBOLS) == names
    others = set(capi.SYMBOLS) | set(capi.SUB_SYMBOLS) | set(capi.FACING_SYMBOLS) | set(capi.RING_SYMBOLS)
    assert not set(capi.SUB_SHARDED_SYMBOLS) & others


def test_null_engine_is_an_error():
    code = '''
import ctypes as C, sys
sys.path.insert(0, %r)
from channeld_b200 import capi
L = capi.lib()
b = capi.SubBatch(n=0)
print("ST", L.chd_apply_subscriptions_sharded(None, C.byref(b), 0, None), L.chd_apply_subscriptions_sharded(None, None, 0, None))
''' % ROOT
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "ST 1 1" in out.stdout, out.stdout


def test_entry_point_declares_the_needs_and_rules_of_the_whole_world_call():
    bodies = _bodies()
    body = bodies[ENTRY]
    enters = re.findall(r"\bCHD_ENTER\s*\(\s*e\s*,([^;]*)\)\s*;", body)
    assert len(enters) == 1
    assert _flags(enters[0]) == _flags("LOCK|COPY_WAIT|FETCH_GUARD") == _flags(NEEDS["chd_apply_subscriptions"])
    via = {n for n, b in bodies.items() if n.startswith("chd_rule_") and _chain_variants(b)}
    assert _chain_variants(body, via) == {ALWAYS}
    assert re.search(r"\bchd_rule_rings_staged\s*\(", body)
    # one implementation behind both calls, each with its slab flag
    assert re.search(r"\breturn\s+apply\s*\([^;]*\btrue\s*\)\s*;", body)
    assert re.search(r"\breturn\s+apply\s*\([^;]*\bfalse\s*\)\s*;", bodies["chd_apply_subscriptions"])


# ---------------------------------------------------------------------------------------------------- route_sub_ops / merge
def _table():
    from channeld_b200 import sharding

    t = sharding.SlotTable(3)
    for j, r in ((10, 0), (11, 1), (12, 2), (13, 1)):
        t.place(j, r)
    for r in range(3):  # one server key per rank
        t.place(("server", 7, r), r)
    return t


def test_route_keeps_array_order_within_each_rank():
    from channeld_b200 import sharding

    t = _table()
    keys = [11, 10, 13, 11, 12, 10, 13]
    routes = sharding.route_sub_ops(t, keys)
    assert len(routes) == 3
    idx = [r[0].tolist() for r in routes]
    assert idx == [[1, 5], [0, 2, 3, 6], [4]]
    for r, (i, s) in enumerate(routes):
        assert s.dtype == np.uint32
        assert s.tolist() == [t.slot[keys[k]] for k in i]
        assert all(t.owner[keys[k]] == r for k in i)


def test_merge_puts_statuses_back_and_unknown_keys_get_err_slot():
    from channeld_b200 import capi, sharding

    t = _table()
    keys = [99, 10, 12, "nobody", 11, 10]
    routes = sharding.route_sub_ops(t, keys)
    assert sum(len(i) for i, _ in routes) == 4
    statuses = [np.array([capi.SUB_NEW, capi.SUB_MERGED], np.uint8), np.array([capi.SUB_UNSUBSCRIBED], np.uint8),
                np.array([capi.SUB_ERR_OUTSIDE_SLAB], np.uint8)]
    got = sharding.merge_sub_status(routes, statuses, len(keys))
    assert got.dtype == np.uint8
    assert got.tolist() == [capi.SUB_ERR_SLOT, capi.SUB_NEW, capi.SUB_ERR_OUTSIDE_SLAB, capi.SUB_ERR_SLOT, capi.SUB_UNSUBSCRIBED, capi.SUB_MERGED]
    empty = sharding.route_sub_ops(t, [])
    assert [len(i) for i, _ in empty] == [0, 0, 0]
    assert len(sharding.merge_sub_status(empty, [np.zeros(0, np.uint8)] * 3, 0)) == 0


def test_a_server_key_per_rank_routes_each_cell_to_the_owner_of_its_column():
    """A server whose ops span every rank's columns: each op names the key of the rank that owns the cell's column."""
    from channeld_b200 import sharding

    t = _table()
    cols, rows, world = 12, 3, 3
    cells = np.arange(cols * rows)
    owner = sharding.owner_of_column(cells % cols, cols, world)
    keys = [("server", 7, int(r)) for r in owner]
    routes = sharding.route_sub_ops(t, keys)
    for r, (i, s) in enumerate(routes):
        lo, hi = sharding.slab_columns(cols, world, r)
        col = cells[i] % cols
        assert len(i) == rows * (hi - lo) and ((col >= lo) & (col < hi)).all()
        assert (s == t.slot[("server", 7, r)]).all()
