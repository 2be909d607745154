"""CPU-side checks of byte-carrying device rings (include/chd_gpu_ring_bytes.h): the header is plain C99 after chd_gpu.h, the library
exports what it declares, a NULL engine is refused everywhere, the entry points declare their needs and apply rules 12 and 13 where
the inventory below says, and the restatement of the byte rule the GPU tests compare against (tests/_ring_bytes.py) gives the
hand-derived results.  No GPU needed."""
import os
import re
import subprocess
import sys

from tests._ring_bytes import MS, ByteRing, msg_indices, update_bytes
from tests.test_entry_points import ALWAYS, NEEDS, _bodies, _chain_variants, _flags

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "chd_gpu_ring_bytes.h")
# the CHD_ENTER of each entry point: the reserve and the append as chd_rings_init / chd_rings_append (the device alone), the
# read-back as chd_get_rings (after the copy wait)
RING_BYTES_NEEDS = {"chd_rings_reserve_bytes": "DEVICE", "chd_rings_append_bytes": "DEVICE", "chd_get_ring_bytes": "COPY_WAIT"}
RING_BYTES_CHAIN = {"chd_rings_reserve_bytes": ALWAYS, "chd_rings_append_bytes": ALWAYS}  # rule 13
RING_BYTES_STAGED = {"chd_rings_reserve_bytes", "chd_rings_append_bytes", "chd_get_ring_bytes"}  # rule 12


def _uncommented():
    return re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)


def _declared():
    return sorted(set(re.findall(r"\b(chd_[a-z0-9_]+)\s*\(", _uncommented())))


def test_header_is_plain_c(tmp_path):
    src = tmp_path / "ring_bytes_hdr.c"
    src.write_text('#include "chd_gpu.h"\n#include "chd_gpu_ring_bytes.h"\n#include "chd_gpu_ring_bytes.h"\n'
                   "int main(void) { chd_status (*f)(chd_engine*, uint32_t) = chd_rings_reserve_bytes;\n"
                   "  chd_status (*g)(chd_engine*, const uint32_t*, uint32_t, const int64_t*, const uint32_t*, const uint64_t*, const uint8_t*) =\n"
                   "      chd_rings_append_bytes;\n"
                   "  chd_status (*h)(chd_engine*, uint64_t*, uint8_t*, uint64_t, uint64_t*) = chd_get_ring_bytes;\n"
                   "  return f == 0 || g == 0 || h == 0; }\n")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src), "-c", "-o",
                           str(tmp_path / "ring_bytes_hdr.o")])


def test_library_exports_every_declared_symbol():
    from channeld_b200 import capi

    L = capi.lib()
    names = _declared()
    for n in names:
        assert hasattr(L, n), "libchd_b200.so does not export %s" % n
    assert sorted(capi.RING_BYTES_SYMBOLS) == names
    others = set(capi.SYMBOLS) | set(capi.SUB_SYMBOLS) | set(capi.FACING_SYMBOLS) | set(capi.RING_SYMBOLS) | set(capi.SUB_SHARDED_SYMBOLS)
    assert not set(capi.RING_BYTES_SYMBOLS) & others


def test_null_engine_is_an_error_everywhere():
    code = '''
import ctypes as C, sys
sys.path.insert(0, %r)
from channeld_b200 import capi
L = capi.lib()
bad = []
for name in capi.RING_BYTES_SYMBOLS:
    f = getattr(L, name)
    assert f.argtypes is not None, name
    args = [None if (t is C.c_void_p or hasattr(t, "contents")) else 0 for t in f.argtypes]
    if f(*args) != capi.ERR_INVALID:
        bad.append(name)
off, boff, t = (C.c_uint32 * 2)(), (C.c_uint64 * 2)(), C.c_uint64()
if L.chd_rings_reserve_bytes(None, 64) != capi.ERR_INVALID:
    bad.append("chd_rings_reserve_bytes(NULL, 64)")
if L.chd_rings_append_bytes(None, off, 0, None, None, boff, None) != capi.ERR_INVALID:
    bad.append("chd_rings_append_bytes(NULL, offsets)")
if L.chd_get_ring_bytes(None, boff, None, 0, C.byref(t)) != capi.ERR_INVALID:
    bad.append("chd_get_ring_bytes(NULL, total)")
print("BAD", bad)
''' % ROOT
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "BAD []" in out.stdout, out.stdout


def test_entry_points_declare_their_needs_and_rules():
    assert set(RING_BYTES_NEEDS) == set(_declared()) and not set(RING_BYTES_NEEDS) & set(NEEDS)
    bodies = _bodies()
    via = {n for n, b in bodies.items() if n.startswith("chd_rule_") and _chain_variants(b)}
    for name, want in RING_BYTES_NEEDS.items():
        body = bodies[name]
        enters = re.findall(r"\bCHD_ENTER\s*\(\s*e\s*,([^;]*)\)\s*;", body)
        assert len(enters) == 1, "%s: %d CHD_ENTER" % (name, len(enters))
        assert _flags(enters[0]) == _flags(want), name
        chain = _chain_variants(body, via)
        assert chain == ({RING_BYTES_CHAIN[name]} if name in RING_BYTES_CHAIN else set()), (name, chain)
        staged = re.search(r"\bchd_rule_rings_staged\s*\(\s*e\s*,", body) is not None
        assert staged == (name in RING_BYTES_STAGED), name
        # every rule is checked before the engine is entered: a refused call changes nothing
        first_enter = body.index("CHD_ENTER")
        assert all(m.start() < first_enter for m in re.finditer(r"\bchd_rule_\w+\s*\(", body)), name
    # rule 14's two append modes: each append entry point refuses the other mode
    assert re.search(r"\bchd_rule_ring_append\s*\(\s*e\s*,\s*true\s*\)", bodies["chd_rings_append_bytes"])
    assert re.search(r"\bchd_rule_ring_append\s*\(\s*e\s*,\s*false\s*\)", bodies["chd_rings_append"])
    assert re.search(r"\bchd_rule_ring_bytes_reserve\s*\(\s*e\s*\)", bodies["chd_rings_reserve_bytes"])
    assert re.search(r"\bchd_rule_assemble_rings\s*\(\s*e\s*\)", bodies["chd_assemble_payloads"])
    assert re.search(r"\bchd_rule_payload_entries\s*\(\s*e\s*,", bodies["chd_set_payload_bytes"])


def _ring(cap, bcap, items, max_iv=0):
    r = ByteRing(cap, bcap)
    dropped = [r.append(t, 1, d, max_iv) for t, d in items]
    return r, dropped


def test_byte_rule_drops_then_slides():
    # 40 + 40 live, then 30: 110 > 100 drops the oldest (CHD_OVF_RING); 80 + 30 > 100 at the tail slides the 40 live bytes by 40
    r, dropped = _ring(513, 100, [(1, b"a" * 40), (2, b"b" * 40), (3, b"c" * 30)])
    assert dropped == [0, 0, 1] and r.drops == 1 and r.byte_slides == [40]
    assert [x[2] for x in r.ents] == [2, 3] and r.mi == 3 and (r.bb, r.be) == (0, 70) and (r.b, r.e) == (1, 3)


def test_byte_rule_slide_shorter_than_a_warp():
    # 530 one-byte entries: from the 513th on the 512 rule (maxFanOutIntervalMs 0) evicts one per update, so 18 bytes are released;
    # then 480 bytes: 512 + 480 <= 1000 fit, but 530 + 480 > 1000 at the tail: a slide by 18 bytes
    items = [(t, b"x") for t in range(1, 531)] + [(531, b"y" * 480)]
    r, dropped = _ring(1024, 1000, items)
    assert sum(dropped) == 0 and r.byte_slides == [18] and r.evictions == 19
    assert len(r.ents) == 512 and r.mi == 531 and (r.bb, r.be) == (1, 992) and r.live_bytes() == 991
    assert r.ents[0][2] == 20 and r.ents[-1][3] == b"y" * 480


def test_byte_rule_empty_updates_and_the_interval():
    # empty updates take entries and no bytes; arrivals within maxFanOutIntervalMs (50 ms) of the newest are kept past 512
    items = [(t * 1000, b"") for t in range(600)]
    r, dropped = _ring(1024, 16, items, max_iv=50)
    assert sum(dropped) == 0 and r.evictions == 0 and len(r.ents) == 600 and r.live_bytes() == 0 and r.byte_slides == []
    # one arrival far in the future: the oldest entry is older than the interval, one eviction per update
    r.append(10_000 * MS, 1, b"zz", 50)
    assert r.evictions == 1 and len(r.ents) == 600 and r.live_bytes() == 2


def test_byte_rule_full_entry_slab():
    # a 513-entry slab that the 512 rule never evicts from (arrivals within the interval): the 514th update finds it full, drops
    # the oldest entry and its bytes, and slides
    items = [(t, bytes([t & 0xFF])) for t in range(514)]
    r, dropped = _ring(513, 4096, items, max_iv=1000)
    assert dropped[-1] == 1 and sum(dropped) == 1 and r.slides == 1 and r.evictions == 0
    assert len(r.ents) == 513 and (r.b, r.e) == (0, 513) and r.ents[0][2] == 2 and r.live_bytes() == 513


def test_update_bytes_follow_the_msg_index():
    cell, idx = msg_indices([0, 3, 3, 5], [10, 0, 7])
    assert cell.tolist() == [0, 0, 0, 2, 2] and idx.tolist() == [11, 12, 13, 8, 9]
    off, data = update_bytes(cell, idx)
    assert off[0] == 0 and len(data) == off[-1] and (off[1:] - off[:-1] <= 23).all()
    off2, data2 = update_bytes(cell[3:], idx[3:])
    assert bytes(data2) == bytes(data[int(off[3]):])
