"""Batched results into device memory (vo_batch_wait_device): the ctypes struct is vo_batch_dresults of the public header
field for field and offset for offset, the entry point is declared, bound with the argument count of its prototype and
exported, and the torch binding refuses bad arguments before any library call."""
import ctypes as C
import os
import re

import pytest

from visual_odom_b200 import capi

torch = pytest.importorskip("torch")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "vo_b200.h")).read()


def test_dresults_struct_matches_the_header():
    body = re.search(r"typedef struct vo_batch_dresults \{(.*?)\} vo_batch_dresults;", HEADER, re.S).group(1)
    fields = re.findall(r"^\s*([\w ]+?)\s*(\*?)\s*(\w+);", body, re.M)
    names = [f[2] for f in fields]
    assert names == [f[0] for f in capi.VoBatchDResults._fields_] == ["records", "pts_cap", "pts4", "kept_idx", "points3d",
                                                                       "inliers", "mono", "ess_mask"]
    for (ctype, star, name), (_, ct) in zip(fields, capi.VoBatchDResults._fields_):
        if star:
            assert ct is C.c_void_p, name
        else:
            assert (ctype, ct) == ("int", C.c_int), name
    # x86-64 / aarch64 C layout: 8-byte pointers, pts_cap padded to the next pointer
    offsets = [getattr(capi.VoBatchDResults, n).offset for n in names]
    assert offsets == [0, 8, 16, 24, 32, 40, 48, 56]
    assert C.sizeof(capi.VoBatchDResults) == 64


def test_entry_point_is_declared_bound_and_exported(built):
    m = re.search(r"VO_API int\s+vo_batch_wait_device\(([^)]*)\);", HEADER)
    assert m, "vo_batch_wait_device is not declared in include/vo_b200.h"
    assert len(m.group(1).split(",")) == 4
    res, args = capi.SIGNATURES["vo_batch_wait_device"]
    assert res is C.c_int and len(args) == 4
    assert args[3]._type_ is capi.VoBatchDResults
    lib = C.CDLL(capi.LIB_PATH)
    assert hasattr(lib, "vo_batch_wait_device"), f"vo_batch_wait_device is not exported by {capi.LIB_PATH}"


class _NoLibrary:
    """Stands in for the loaded library: any entry point reached is a failure of the binding's own checks."""
    def __getattr__(self, name):
        raise AssertionError(f"the binding called {name}")


def _context():
    c = object.__new__(capi.Context)
    c.h, c.device, c.lib = None, 0, _NoLibrary()
    return c


@pytest.mark.parametrize("cap", [0, -1, 2.5, None])
def test_lists_without_a_capacity_are_refused(cap):
    c = _context()
    with pytest.raises(ValueError, match="pts_cap"):
        c.batch_wait_device(0, 4, pts_cap=cap)
    with pytest.raises(ValueError, match="pts_cap"):
        c.batch_wait_device(0, 4, pts_cap=cap, points=False, points3d=False, inliers=False)      # kept_idx alone
    with pytest.raises(ValueError, match="pts_cap"):
        c.batch_dresults_alloc(4, pts_cap=cap, points=False, kept_idx=False, points3d=False, inliers=False, mono=True)
    # an out= dict with a list and no (or a bad) pts_cap
    bad = dict(kept_idx=torch.zeros((4, 0), dtype=torch.int32))
    if cap is not None:
        bad["pts_cap"] = cap
    with pytest.raises(ValueError, match="pts_cap"):
        c.batch_wait_device(0, 4, out=bad)


def test_out_tensors_must_be_cuda_tensors():
    c = _context()
    with pytest.raises(TypeError, match="CUDA"):
        c.batch_wait_device(0, 3, out=dict(pts_cap=16, records=torch.zeros((3, 19), dtype=torch.float64)))
    with pytest.raises(TypeError, match="CUDA"):
        c.batch_wait_device(0, 3, out=dict(pts_cap=16, kept_idx=torch.zeros((3, 16), dtype=torch.int32)))
    with pytest.raises(TypeError, match="CUDA"):
        c.batch_wait_device(0, 3, out=dict(pts_cap=16, inliers=[0] * 48))


def test_out_shapes_and_dtypes_are_checked():
    c = _context()
    for bad in (dict(pts_cap=16, records=torch.zeros((2, 19), dtype=torch.float64)),          # not the submission's count
                dict(pts_cap=16, records=torch.zeros((3, 19), dtype=torch.float32)),
                dict(pts_cap=16, kept_idx=torch.zeros((3, 8), dtype=torch.int32)),             # not pts_cap
                dict(pts_cap=16, kept_idx=torch.zeros((3, 16), dtype=torch.int64)),
                dict(pts_cap=16, pts4=torch.zeros((3, 4, 8, 2), dtype=torch.float32)),
                dict(pts_cap=16, points3d=torch.zeros((3, 16, 3), dtype=torch.float64)),
                dict(pts_cap=16, ess_mask=torch.zeros((3, 16), dtype=torch.bool)),
                dict(pts_cap=16, mono_raw=torch.zeros((3, 14), dtype=torch.float64).t().contiguous().t())):
        with pytest.raises(ValueError, match="out"):
            c.batch_wait_device(0, 3, out=bad)


def test_timing_tool_check_runs_without_a_gpu():
    import json
    import subprocess
    import sys
    tool = os.path.join(ROOT, "tools", "batch_device_results_timing.py")
    out = subprocess.run([sys.executable, tool, "--check", "--rounds", "3", "--seconds", "1"], capture_output=True, text=True,
                         timeout=120)
    assert out.returncode == 0, out.stderr
    p = json.loads(out.stdout)["plan"]
    assert p["modes"] == ["host+lists", "host", "device"] and p["in_flight"] == 3 and p["units_per_submission"] == 8
    assert p["size"] == [1241, 376] and p["features"] == 2000
    bad = subprocess.run([sys.executable, tool, "--check", "--rounds", "2"], capture_output=True, text=True, timeout=120)
    assert bad.returncode != 0
