"""CPU-side checks of ring limits across slabs (include/chd_gpu_rings.h): the header is plain C99 next to chd_gpu.h, the library exports
what it declares, and every entry point refuses a NULL engine.  No GPU needed."""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "chd_gpu_rings.h")


def _uncommented():
    return re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)


def _declared():
    return sorted(set(re.findall(r"\b(chd_[a-z0-9_]+)\s*\(", _uncommented())))


def test_header_is_plain_c(tmp_path):
    src = tmp_path / "rings_hdr.c"
    src.write_text('#include "chd_gpu.h"\n#include "chd_gpu_rings.h"\n#include "chd_gpu_rings.h"\n'
                   "int main(void) { chd_status (*f)(chd_engine*, uint32_t*, uint32_t, uint32_t*) = chd_export_ring_limits;\n"
                   "  chd_status (*g)(chd_engine*, const uint32_t*, uint32_t) = chd_import_ring_limits; return f == 0 || g == 0; }\n")
    exe = tmp_path / "rings_hdr"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src), "-c", "-o",
                           str(exe) + ".o"])


def test_library_exports_every_declared_symbol():
    from channeld_b200 import capi

    L = capi.lib()
    names = _declared()
    for n in names:
        assert hasattr(L, n), "libchd_b200.so does not export %s" % n
    assert sorted(capi.RING_SYMBOLS) == names
    assert not set(capi.RING_SYMBOLS) & (set(capi.SYMBOLS) | set(capi.SUB_SYMBOLS) | set(capi.FACING_SYMBOLS))


def test_null_engine_is_an_error_everywhere():
    code = '''
import ctypes as C, sys
sys.path.insert(0, %r)
from channeld_b200 import capi
L = capi.lib()
bad = []
for name in capi.RING_SYMBOLS:
    f = getattr(L, name)
    assert f.argtypes is not None, name
    args = [None if (t is C.c_void_p or hasattr(t, "contents")) else 0 for t in f.argtypes]
    if f(*args) != capi.ERR_INVALID:
        bad.append(name)
n = C.c_uint32()
if L.chd_export_ring_limits(None, None, 0, C.byref(n)) != capi.ERR_INVALID:
    bad.append("chd_export_ring_limits(NULL, count)")
print("BAD", bad)
''' % ROOT
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "BAD []" in out.stdout, out.stdout
