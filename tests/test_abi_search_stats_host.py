"""Host-side check that needs no GPU: api.SearchStats mirrors lb200_search_stats_t field for field, as the C compiler lays it out."""
import ctypes as C
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_search_stats_layout_matches_header(tmp_path):
    from lantern_b200 import api
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    fields = [f for f, _ in api.SearchStats._fields_]
    src = ['#include <stddef.h>', '#include <stdio.h>', '#include "lantern_b200.h"', "int main(void) {",
           '    printf("%zu\\n", sizeof(lb200_search_stats_t));']
    src += ['    printf("%%zu\\n", offsetof(lb200_search_stats_t, %s));' % f for f in fields]
    src += ["    return 0;", "}"]
    (tmp_path / "layout.c").write_text("\n".join(src) + "\n")
    exe = str(tmp_path / "layout")
    subprocess.check_call([cc, "-std=c11", "-I", os.path.join(ROOT, "include"), str(tmp_path / "layout.c"), "-o", exe])
    got = [int(v) for v in subprocess.check_output([exe]).split()]
    assert got[0] == C.sizeof(api.SearchStats)
    assert got[1:] == [getattr(api.SearchStats, f).offset for f in fields]
    assert fields[-6:] == ["search_kernel", "reserved", "owner_cycles_produce", "owner_cycles_screen", "owner_cycles_evaluate",
                           "owner_cycles_consume"]
