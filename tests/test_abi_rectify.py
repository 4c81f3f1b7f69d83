"""Rectification's C-ABI without a GPU: vo_rectify_maps, vo_remap, vo_seq_rectify and vo_mseq_rectify are declared,
bound with their prototypes' argument counts and exported; vo_rectify_cam / vo_rectify keep the header's layout field for
field; vo_rectify_maps refuses what it documents (n_d not 4, 5 or 8, a non-finite entry, a singular P * R, a size <= 0,
NULL pointers) and writes nothing then."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from visual_odom_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "vo_b200.h")).read()
SYMBOLS = {"vo_rectify_maps": 5, "vo_remap": 9, "vo_seq_rectify": 2, "vo_mseq_rectify": 4}


def test_entry_points_are_declared_bound_and_exported(built):
    lib = C.CDLL(capi.LIB_PATH)
    for name, nargs in SYMBOLS.items():
        m = re.search(r"VO_API int\s+" + name + r"\(([^)]*)\);", HEADER)
        assert m, f"{name} is not declared in include/vo_b200.h"
        assert len(m.group(1).split(",")) == nargs
        assert name in capi.SIGNATURES and len(capi.SIGNATURES[name][1]) == nargs
        assert hasattr(lib, name), f"{name} is not exported"


def test_struct_layout_is_the_headers():
    body = re.search(r"typedef struct vo_rectify_cam \{(.*?)\} vo_rectify_cam;", HEADER, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = re.findall(r"^\s*(int|double)\s+(\w+)(?:\[(\d+)\])?\s*;", body, re.M)
    assert [f[1] for f in fields] == [f[0] for f in capi.VoRectifyCam._fields_] == ["K", "D", "n_d", "R", "P"]
    assert [int(f[2] or 1) for f in fields] == [9, 8, 1, 9, 9]
    assert capi.VoRectifyCam.n_d.offset == 136 and capi.VoRectifyCam.R.offset == 144 and C.sizeof(capi.VoRectifyCam) == 288
    assert re.search(r"typedef struct vo_rectify \{ vo_rectify_cam left, right; \} vo_rectify;", HEADER)
    assert capi.VoRectify.right.offset == 288 and C.sizeof(capi.VoRectify) == 576


GOOD = (np.array([[458.654, 0, 367.215], [0, 457.296, 248.375], [0, 0, 1]]),
        np.array([-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05, 0.0]), np.eye(3),
        np.array([[435.2, 0, 367.45, 0], [0, 435.2, 252.2, 0], [0, 0, 1, 0]]))


def _maps(c, w=16, h=8):
    lib = capi.load_library()
    mx = np.full((max(h, 1), max(w, 1)), -7.0, np.float32)
    my = mx.copy()
    rc = lib.vo_rectify_maps(C.byref(c), w, h, mx.ctypes.data_as(C.c_void_p), my.ctypes.data_as(C.c_void_p))
    return rc, mx, my


def test_refusals_of_vo_rectify_maps(built):
    rc, mx, _ = _maps(capi.rectify_cam(*GOOD))
    assert rc == capi.VO_OK and (mx != -7.0).all()
    bad = []
    for n_d in (0, 3, 6, 7, 9):
        c = capi.rectify_cam(*GOOD); c.n_d = n_d; bad.append(c)
    for field, i in (("K", 0), ("K", 8), ("R", 4), ("P", 2)):
        for v in (float("nan"), float("inf"), -float("inf")):
            c = capi.rectify_cam(*GOOD); getattr(c, field)[i] = v; bad.append(c)
    c = capi.rectify_cam(*GOOD); c.D[4] = float("nan"); bad.append(c)
    c = capi.rectify_cam(*GOOD); c.P[:] = [1, 0, 0, 0, 1, 0, 0, 0, 0]; bad.append(c)           # singular P
    c = capi.rectify_cam(*GOOD); c.R[:] = [1, 0, 0, 2, 0, 0, 0, 0, 1]; bad.append(c)           # singular R
    for c in bad:
        rc, mx, my = _maps(c)
        assert rc == capi.VO_E_INVALID and (mx == -7.0).all() and (my == -7.0).all()
    # a NaN coefficient past n_d is not read
    c = capi.rectify_cam(*GOOD); c.n_d = 4; c.D[4] = float("nan")
    assert _maps(c)[0] == capi.VO_OK
    lib = capi.load_library()
    good = capi.rectify_cam(*GOOD)
    for w, h in ((0, 8), (16, 0), (-1, 8)):
        assert _maps(good, w, h)[0] == capi.VO_E_INVALID
    buf = np.zeros(128, np.float32)
    assert lib.vo_rectify_maps(None, 16, 8, buf.ctypes.data_as(C.c_void_p), buf.ctypes.data_as(C.c_void_p)) == capi.VO_E_INVALID
    assert lib.vo_rectify_maps(C.byref(good), 16, 8, None, buf.ctypes.data_as(C.c_void_p)) == capi.VO_E_INVALID


def test_rectify_cam_takes_the_settings_files_shapes():
    c = capi.rectify_cam(*GOOD)
    assert c.n_d == 5 and list(c.P) == [435.2, 0, 367.45, 0, 435.2, 252.2, 0, 0, 1]
    with pytest.raises(ValueError):
        capi.rectify_cam(GOOD[0], np.zeros(9), GOOD[2], GOOD[3])
