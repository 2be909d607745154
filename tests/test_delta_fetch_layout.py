"""CPU-side check of the visible-delta read-back structs: chd_delta_buffers and chd_delta_counts have the size and field offsets in
ctypes (channeld_b200/capi.py) that gcc gives them in include/chd_gpu.h.  Runs without a GPU."""
import ctypes as C
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_delta_structs_match_header(tmp_path):
    from channeld_b200 import capi

    pairs = [("chd_delta_buffers", capi.DeltaBuffers), ("chd_delta_counts", capi.DeltaCounts)]
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
    assert C.sizeof(capi.DeltaBuffers) == 6 * 8 and C.sizeof(capi.DeltaCounts) == 3 * 8
