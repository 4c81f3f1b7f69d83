"""The entry points that start sequences in a running multi-sequence context are exported, declared in the public header
and bound in capi.SIGNATURES with the argument counts of their prototypes, and capi.VoMseqStart has the size and field
offsets of the C struct vo_mseq_start as the host compiler lays it out."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = {"vo_mseq_open": 5, "vo_mseq_submit_start": 7}


def test_start_entry_points_are_declared_bound_and_exported(built):
    import ctypes as C
    from visual_odom_b200 import capi
    header = open(os.path.join(ROOT, "include", "vo_b200.h")).read()
    lib = C.CDLL(capi.LIB_PATH)
    for name, nargs in SYMBOLS.items():
        m = re.search(r"VO_API int " + name + r"\(([^)]*)\);", header)
        assert m, f"{name} is not declared in include/vo_b200.h"
        assert len(m.group(1).split(",")) == nargs
        assert name in capi.SIGNATURES and len(capi.SIGNATURES[name][1]) == nargs
        assert hasattr(lib, name), f"{name} is not exported by {capi.LIB_PATH}"
    m = re.search(r"#define VO_MSEQ_STARTED (\d+)", header)
    assert m and int(m.group(1)) == capi.VO_MSEQ_STARTED
    assert capi.VO_MSEQ_STARTED not in (capi.VO_OK, capi.VO_MSEQ_RETIRED)


def test_the_start_record_matches_the_c_layout(tmp_path):
    import ctypes as C
    from visual_odom_b200 import capi
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no host C compiler")
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "vo_b200.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(vo_mseq_start), offsetof(vo_mseq_start, slot),\n'
                   '         offsetof(vo_mseq_start, w), offsetof(vo_mseq_start, h), offsetof(vo_mseq_start, P_l),\n'
                   '         offsetof(vo_mseq_start, P_r));\n  return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    S = capi.VoMseqStart
    assert got == [C.sizeof(S), S.slot.offset, S.w.offset, S.h.offset, S.P_l.offset, S.P_r.offset]
