"""Device-image descriptors without a GPU: what capi.image_descriptor derives from a tensor's shape and strides, what it
refuses, and the ctypes layout of vo_dimage / vo_dunit against the header (compiled with the host compiler)."""
import ctypes as C
import os
import shutil
import subprocess
import types

import numpy as np
import pytest

from visual_odom_b200 import capi

torch = pytest.importorskip("torch")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def desc(t, order=None):
    d, w, h = capi.image_descriptor(t.shape, t.stride(), t.data_ptr(), order)
    return (d.data - t.data_ptr(), d.row_pitch, d.pixel_stride, d.channel_stride, d.format, w, h)


def test_gray_hwc_chw():
    h, w = 7, 13
    assert desc(torch.zeros(h, w, dtype=torch.uint8)) == (0, w, 1, 0, capi.VO_FMT_GRAY, w, h)
    assert desc(torch.zeros(h, w, 3, dtype=torch.uint8), "bgr") == (0, 3 * w, 3, 1, capi.VO_FMT_BGR, w, h)
    assert desc(torch.zeros(h, w, 3, dtype=torch.uint8), "rgb") == (0, 3 * w, 3, 1, capi.VO_FMT_RGB, w, h)
    assert desc(torch.zeros(3, h, w, dtype=torch.uint8), "rgb") == (0, w, 1, h * w, capi.VO_FMT_RGB, w, h)


def test_column_slice_of_a_wider_tensor():
    """Odd base offset and a row pitch other than the width: the descriptor points at the slice, the pitch stays the
    wider tensor's."""
    big = torch.zeros(9, 40, 3, dtype=torch.uint8)
    t = big[2:, 3:3 + 31]
    d, w, h = capi.image_descriptor(t.shape, t.stride(), t.data_ptr(), "bgr")
    assert d.data - big.data_ptr() == 2 * 120 + 9                  # odd
    assert (d.row_pitch, d.pixel_stride, d.channel_stride, w, h) == (120, 3, 1, 31, 7)
    g = torch.zeros(8, 1243, dtype=torch.uint8)[:, 1:1 + 1241]
    d, w, h = capi.image_descriptor(g.shape, g.stride(), g.data_ptr())
    assert (d.data - g.data_ptr(), d.row_pitch, d.pixel_stride, w, h) == (0, 1243, 1, 1241, 8)
    c = torch.zeros(3, 6, 50, dtype=torch.uint8)[:, 1:, 5:46]      # planar crop
    assert desc(c, "bgr") == (0, 50, 1, 300, capi.VO_FMT_BGR, 41, 5)


def test_transposed_and_negative_stride_images_are_refused():
    t = torch.zeros(11, 5, dtype=torch.uint8).t()                   # (5, 11) with strides (1, 5): rows overlap
    with pytest.raises(ValueError, match="overlap"):
        capi.image_descriptor(t.shape, t.stride(), t.data_ptr())
    a = np.zeros((4, 6), np.uint8)[:, ::-1]                         # numpy byte strides (6, -1)
    with pytest.raises(ValueError, match="positive"):
        capi.image_descriptor(a.shape, a.strides, a.ctypes.data)
    e = torch.zeros(1, 6, dtype=torch.uint8).expand(4, 6)           # zero row stride
    with pytest.raises(ValueError, match="positive"):
        capi.image_descriptor(e.shape, e.stride(), e.data_ptr())


def test_colour_needs_an_order_and_an_unambiguous_layout():
    with pytest.raises(ValueError, match="order"):
        desc(torch.zeros(4, 5, 3, dtype=torch.uint8))
    with pytest.raises(ValueError, match="order"):
        desc(torch.zeros(4, 5, 3, dtype=torch.uint8), "gray")
    with pytest.raises(ValueError, match="expected"):
        desc(torch.zeros(3, 5, 3, dtype=torch.uint8), "bgr")
    with pytest.raises(ValueError, match="expected"):
        desc(torch.zeros(4, 5, 4, dtype=torch.uint8), "bgr")
    with pytest.raises(ValueError, match="expected"):
        desc(torch.zeros(2, 4, 5, 3, dtype=torch.uint8), "bgr")


def test_cpu_tensors_and_other_dtypes_are_refused_before_the_library():
    fake = types.SimpleNamespace(device=0)                          # no context (and no GPU) needed for the checks
    with pytest.raises(TypeError, match="CUDA"):
        capi.Context._device_image(fake, torch.zeros(4, 5, dtype=torch.uint8), None)
    with pytest.raises(TypeError, match="CUDA"):
        capi.Context._device_image(fake, np.zeros((4, 5), np.uint8), None)


def test_struct_layout_matches_the_header(tmp_path):
    if not shutil.which("g++"):
        pytest.skip("no host C++ compiler")
    src = tmp_path / "layout.cpp"
    src.write_text(r'''
#include <cstdio>
#include <cstddef>
#include "vo_b200.h"
#define F(T, f) std::printf(#T "." #f " %zu\n", offsetof(T, f));
int main() {
    std::printf("vo_dimage %zu\nvo_dunit %zu\n", sizeof(vo_dimage), sizeof(vo_dunit));
    F(vo_dimage, data) F(vo_dimage, row_pitch) F(vo_dimage, pixel_stride) F(vo_dimage, channel_stride) F(vo_dimage, format)
    F(vo_dunit, l0) F(vo_dunit, r0) F(vo_dunit, l1) F(vo_dunit, r1) F(vo_dunit, pts) F(vo_dunit, n_pts) F(vo_dunit, t_prev)
    std::printf("fmt %d %d %d\n", VO_FMT_GRAY, VO_FMT_BGR, VO_FMT_RGB);
}
''')
    exe = tmp_path / "layout"
    subprocess.run(["g++", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = dict(ln.split(" ", 1) for ln in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["vo_dimage"]) == C.sizeof(capi.VoDImage)
    assert int(got["vo_dunit"]) == C.sizeof(capi.VoDUnit)
    for T, name in ((capi.VoDImage, "vo_dimage"), (capi.VoDUnit, "vo_dunit")):
        for f, _ in T._fields_:
            assert int(got[f"{name}.{f}"]) == getattr(T, f).offset, (name, f)
    assert got["fmt"] == f"{capi.VO_FMT_GRAY} {capi.VO_FMT_BGR} {capi.VO_FMT_RGB}"
