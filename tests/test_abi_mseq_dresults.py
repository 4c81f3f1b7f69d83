"""Results into device memory (vo_mseq_wait_device, the flag VO_MSEQ_DEVICE_RESULTS, vo_pose_step_device): the ctypes
struct is vo_mseq_dresults of the public header field for field, the entry points are declared, bound with the argument
counts of their prototypes and exported, the flag has its header value, and the torch binding refuses bad arguments before
any library call."""
import ctypes as C
import os
import re

import pytest

from visual_odom_b200 import capi

torch = pytest.importorskip("torch")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "vo_b200.h")).read()
SYMBOLS = {"vo_mseq_wait_device": 2, "vo_pose_step_device": 6}


def test_dresults_struct_matches_the_header():
    body = re.search(r"typedef struct vo_mseq_dresults \{(.*?)\} vo_mseq_dresults;", HEADER, re.S).group(1)
    fields = re.findall(r"^\s*([\w ]+?)\s*(\*?)\s*(\w+);", body, re.M)
    names = [f[2] for f in fields]
    assert names == [f[0] for f in capi.VoMseqDResults._fields_]
    for (ctype, star, name), (_, ct) in zip(fields, capi.VoMseqDResults._fields_):
        if star:
            assert ct is C.c_void_p, name
        else:
            assert (ctype, ct) == ("int", C.c_int), name
    # pointers are 8 bytes, pts_cap is padded to the next pointer
    assert capi.VoMseqDResults.pts_cap.offset == 24 and capi.VoMseqDResults.pts4.offset == 32
    assert C.sizeof(capi.VoMseqDResults) == 8 * 9


def test_flag_value_and_bit():
    m = re.search(r"#define VO_MSEQ_DEVICE_RESULTS (\d+)", HEADER)
    assert m and int(m.group(1)) == capi.VO_MSEQ_DEVICE_RESULTS == 8
    # a bit of its own: not the mono flag, and not bits 2 or 4, which stay unknown (refused)
    assert capi.VO_MSEQ_DEVICE_RESULTS & (capi.VO_MSEQ_MONO_ROTATION | 2 | 4) == 0


def test_entry_points_are_declared_bound_and_exported(built):
    lib = C.CDLL(capi.LIB_PATH)
    for name, nargs in SYMBOLS.items():
        m = re.search(r"VO_API int\s+" + name + r"\(([^)]*)\);", HEADER)
        assert m, f"{name} is not declared in include/vo_b200.h"
        assert len(m.group(1).split(",")) == nargs
        assert name in capi.SIGNATURES and len(capi.SIGNATURES[name][1]) == nargs
        assert hasattr(lib, name), f"{name} is not exported by {capi.LIB_PATH}"
    assert capi.SIGNATURES["vo_mseq_wait_device"][1][1]._type_ is capi.VoMseqDResults


class _NoLibrary:
    """Stands in for the loaded library: any entry point reached is a failure of the binding's own checks."""
    def __getattr__(self, name):
        raise AssertionError(f"the binding called {name}")


def _context(n=3, mono=False):
    c = object.__new__(capi.Context)
    c.h, c.device, c.lib = None, 0, _NoLibrary()
    c._mseq_n, c._mseq_mono = n, mono
    return c


@pytest.mark.parametrize("cap", [0, -1, 2.5, None])
def test_point_outputs_without_a_capacity_are_refused(cap):
    c = _context()
    with pytest.raises(ValueError, match="pts_cap"):
        c.mseq_wait_device(pts_cap=cap)
    with pytest.raises(ValueError, match="pts_cap"):
        c.mseq_wait_device(pts_cap=cap, points=False, points3d=False)


def test_out_tensors_must_be_cuda_tensors_of_the_run():
    c = _context(3)
    with pytest.raises(TypeError, match="CUDA"):
        c.mseq_wait_device(out=dict(pts_cap=16, status=torch.zeros(3, dtype=torch.int32)))
    with pytest.raises(TypeError, match="CUDA"):
        c.mseq_wait_device(out=dict(pts_cap=16, records=torch.zeros((3, 19), dtype=torch.float64)))


def test_out_shapes_and_dtypes_are_checked():
    c = _context(3)
    for bad in (dict(pts_cap=16, status=torch.zeros(2, dtype=torch.int32)),
                dict(pts_cap=16, status=torch.zeros(3, dtype=torch.int64)),
                dict(pts_cap=16, pts4=torch.zeros((3, 4, 8, 2), dtype=torch.float32)),
                dict(pts_cap=16, points3d=torch.zeros((3, 16, 3), dtype=torch.float64)),
                dict(pts_cap=16, frame_pose=torch.zeros((3, 4, 4), dtype=torch.float64).transpose(1, 2))):
        with pytest.raises(ValueError, match="out"):
            c.mseq_wait_device(out=bad)
    with pytest.raises(TypeError, match="CUDA"):
        c.mseq_wait_device(out=dict(pts_cap=16, inliers=[0] * 48))
