"""The per-sequence image-size entry points of the multi-sequence mode are exported, declared in the public header and
bound in capi.SIGNATURES with the argument counts of their prototypes."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = {"vo_mseq_begin_sized": 11, "vo_mseq_submit_sized": 5}


def test_sized_entry_points_are_declared_bound_and_exported(built):
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
