"""Rectification on the CPU, against cv2 4.13: vo_rectify_maps gives cv2's CV_32FC1 maps bit for bit (EuRoC cam0 / cam1,
a KITTI-raw-like camera, 4- and 8-coefficient cameras, identity D and R, strong barrel distortion, odd sizes and
random cameras); the numpy restatement of remap(INTER_LINEAR, BORDER_CONSTANT
0) gives cv2.remap's bytes on maps that sit on integers and on the k/32 rounding ties, go negative, run past w / h by less
and by more than one pixel and past the int16 range; and the ingest kernel's tap arithmetic (remap_math.cuh compiled for
the host) gives the restatement's bytes.  The stereo settings reader of tools/run_sequence.py reads what
cv2.FileStorage reads."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from visual_odom_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import rectify_ref as rr  # noqa: E402

cv2 = pytest.importorskip("cv2")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CV_CPU_FMA3, CV_CPU_AVX2 = 12, 13          # OpenCV's cv::CpuFeatures

EUROC_CAM0, EUROC_CAM1 = synth.RECTIFY_CAMS["euroc_cam0"], synth.RECTIFY_CAMS["euroc_cam1"]
KITTI_RAW = synth.RECTIFY_CAMS["kitti_raw_left"]
FOUR = dict(K=[500.0, 0, 320.5, 0, 505.0, 240.25, 0, 0, 1], D=[-0.12, 0.03, 0.0004, -0.0002],
            R=np.eye(3).ravel(), P=[480.0, 0, 318.0, 0, 480.0, 242.0, 0, 0, 1])
RATIONAL = dict(K=[600.0, 0, 400.0, 0, 598.0, 300.0, 0, 0, 1],
                D=[0.8, -0.2, 0.001, -0.0015, 0.05, 1.1, -0.1, 0.09],
                R=[0.99995, -0.0087, 0.0049, 0.0087, 0.99996, 0.0012, -0.0049, -0.0012, 0.99999],
                P=[560.0, 0, 402.0, 0, 560.0, 299.0, 0, 0, 1])
IDENTITY = dict(K=[700.0, 0, 620.0, 0, 700.0, 188.0, 0, 0, 1], D=[0, 0, 0, 0, 0], R=np.eye(3).ravel(),
                P=[700.0, 0, 620.0, 0, 700.0, 188.0, 0, 0, 1])
BARREL = dict(K=[400.0, 0, 320.0, 0, 400.0, 240.0, 0, 0, 1], D=[-0.6, 0.45, 0.0, 0.0, -0.2], R=np.eye(3).ravel(),
              P=[250.0, 0, 320.0, 0, 250.0, 240.0, 0, 0, 1])      # maps run far outside the image
CASES = [("euroc_cam0", EUROC_CAM0, 752, 480), ("euroc_cam1", EUROC_CAM1, 752, 480), ("kitti_raw", KITTI_RAW, 1242, 375),
         ("four", FOUR, 640, 480), ("rational", RATIONAL, 800, 600), ("identity", IDENTITY, 1241, 376),
         ("barrel", BARREL, 640, 480), ("odd", EUROC_CAM0, 751, 479), ("odd_small", RATIONAL, 97, 33)]


def _random_cameras(n, seed):
    rng = np.random.default_rng(seed)
    out = []
    for t in range(n):
        k = int(rng.choice([4, 5, 8]))
        D = rng.normal(0, 0.3, k) * np.array([1, 1, 0.01, 0.01, 1, 1, 1, 1][:k])
        R = cv2.Rodrigues(rng.normal(0, 0.02, 3))[0].ravel()
        K = [rng.uniform(200, 900), 0, rng.uniform(100, 700), 0, rng.uniform(200, 900), rng.uniform(100, 400), 0, 0, 1]
        P = [rng.uniform(200, 900), 0, rng.uniform(100, 700), 0, rng.uniform(200, 900), rng.uniform(100, 400), 0, 0, 1]
        out.append((f"random{t}", dict(K=K, D=D, R=R, P=P), int(rng.integers(9, 900)), int(rng.integers(3, 600))))
    return out


CASES += _random_cameras(12, 1)


_mats = synth.rectify_cam_matrices


def _cv2_maps(c, w, h):
    K, D, R, P = _mats(c)
    return cv2.initUndistortRectifyMap(K, D, R, P[:, :3], (w, h), cv2.CV_32FC1)


@pytest.mark.parametrize("name,cam,w,h", CASES, ids=[c[0] for c in CASES])
def test_library_maps_are_cv2s(built, name, cam, w, h):
    from visual_odom_b200 import capi
    if not (cv2.useOptimized() and cv2.checkHardwareSupport(CV_CPU_AVX2) and cv2.checkHardwareSupport(CV_CPU_FMA3)):
        pytest.skip("vo_rectify_maps is cv2's AVX2 build of initUndistortRectifyMap; this cv2 runs another one")
    mx, my = capi.rectify_maps(_mats(cam), w, h)
    cx, cy = _cv2_maps(cam, w, h)
    assert np.array_equal(mx.view(np.uint32), cx.view(np.uint32)) and np.array_equal(my.view(np.uint32), cy.view(np.uint32))
    if name == "barrel":
        assert mx.min() < -20 and mx.max() > w + 20 and my.min() < -20, "the barrel case must leave the image"


def edge_maps(w, h, seed):
    """Random maps with every edge the fixed-point conversion and the border have: integers, k/32 ties, negative
    coordinates, coordinates past w / h by less and by more than one pixel, magnitudes past the int16 range."""
    rng = np.random.default_rng(seed)
    mx = rng.uniform(-3, w + 3, (h, w)).astype(np.float32)
    my = rng.uniform(-3, h + 3, (h, w)).astype(np.float32)
    mx[::7] = np.round(mx[::7]); my[::5] = np.round(my[::5])
    mx[1::9] = (np.floor(mx[1::9] * 32) + 0.5) / 32
    my[2::11] = (np.floor(my[2::11] * 32) + 0.5) / 32
    mx[:, -3:] = w - 1 + rng.uniform(0, 2.5, (h, 3)); my[-3:] = h - 1 + rng.uniform(0, 2.5, (3, w))
    mx[:, :3] = rng.uniform(-2.5, 0.5, (h, 3)); my[:3] = rng.uniform(-2.5, 0.5, (3, w))
    mx[3::13, ::3] = rng.uniform(-1e6, 1e6, mx[3::13, ::3].shape)
    my[4::17, ::5] = rng.uniform(-5e4, 5e4, my[4::17, ::5].shape)
    mx[5::19, 1::4] = rng.choice([32767.5, 32768.0, -32768.5, -32769.0, 40000.0, -40000.0], mx[5::19, 1::4].shape)
    return mx, my


def test_edge_maps_have_their_edges():
    mx, my = edge_maps(301, 77, 0)
    fx = mx * 32
    assert (mx == np.round(mx)).any() and (np.abs(fx - np.floor(fx) - 0.5) == 0).any()
    assert (mx < 0).any() and ((mx > 300) & (mx < 301)).any() and (mx > 301).any() and (my > 77).any()
    assert (np.abs(mx) > 32768).any() and (np.abs(my) > 32768).any()


@pytest.mark.parametrize("w,h,seed", [(1241, 376, 0), (301, 77, 1), (64, 6, 2)])
def test_numpy_remap_is_cv2s(w, h, seed):
    mx, my = edge_maps(w, h, seed)
    src = np.random.default_rng(seed + 10).integers(0, 256, (h, w), dtype=np.uint8)
    want = cv2.remap(src, mx, my, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    assert np.array_equal(rr.remap(src, mx, my), want)
    m1, m2 = cv2.convertMaps(mx, my, cv2.CV_16SC2)
    sx, sy, a = rr.fixed_maps(mx, my)
    assert np.array_equal(m1[..., 0], sx) and np.array_equal(m1[..., 1], sy) and np.array_equal(m2, a)


def test_numpy_remap_of_a_rectification_is_cv2s():
    src = np.random.default_rng(3).integers(0, 256, (480, 640), dtype=np.uint8)
    mx, my = _cv2_maps(BARREL, 640, 480)
    want = cv2.remap(src, mx, my, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    assert np.array_equal(rr.remap(src, mx, my), want)


def test_colour_is_remapped_as_converted_gray():
    bgr = np.random.default_rng(4).integers(0, 256, (90, 130, 3), dtype=np.uint8)
    mx, my = edge_maps(130, 90, 5)
    want = cv2.remap(cv2.cvtColor(bgr, cv2.COLOR_BGR2GRAY), mx, my, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT)
    assert np.array_equal(rr.gray_of(bgr), cv2.cvtColor(bgr, cv2.COLOR_BGR2GRAY))
    assert np.array_equal(rr.remap(rr.gray_of(bgr), mx, my), want)


def test_kernel_tap_arithmetic_is_the_oracles(built):
    from visual_odom_b200 import build
    lib = C.CDLL(build.HOSTCHECK_LIB)
    for w, h, seed in ((1241, 376, 6), (97, 33, 7)):
        mx, my = edge_maps(w, h, seed)
        src = np.random.default_rng(seed).integers(0, 256, (h, w), dtype=np.uint8)
        sx, sy, a = rr.fixed_maps(mx, my)
        xy = np.ascontiguousarray(np.stack([sx, sy], -1))
        out = np.empty((h, w), np.uint8)
        lib.vo_hostcheck_remap(src.ctypes.data_as(C.c_void_p), w, h, xy.ctypes.data_as(C.c_void_p),
                               np.ascontiguousarray(a).ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
        assert np.array_equal(out, rr.remap_fixed(src, sx, sy, a))


def _settings_text(cams, w, h):
    def node(name, a):
        a = np.asarray(a, np.float64)
        rows, cols = (1, a.size) if a.ndim == 1 else a.shape
        vals = ", ".join(repr(float(v)) for v in a.ravel())
        return f"{name}: !!opencv-matrix\n   rows: {rows}\n   cols: {cols}\n   dt: d\n   data: [{vals}]\n"
    out = "%YAML:1.0\n"
    for side, c in zip(("LEFT", "RIGHT"), cams):
        K, D, R, P = _mats(c)
        out += f"{side}.height: {h}\n{side}.width: {w}\n"
        out += node(f"{side}.D", D) + node(f"{side}.K", K) + node(f"{side}.R", R) + node(f"{side}.P", P)
    return out + "Camera.fx: 435.2046959714599\n"


def test_settings_reader_reads_what_cv2_reads(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import run_sequence
    path = tmp_path / "euroc.yaml"
    path.write_text(_settings_text([EUROC_CAM0, EUROC_CAM1], 752, 480))
    got = run_sequence.read_rectify(str(path))
    fs = cv2.FileStorage(str(path), cv2.FILE_STORAGE_READ)
    for side in ("LEFT", "RIGHT"):
        for k, a in zip("KDRP", got[side.lower()]):
            want = fs.getNode(f"{side}.{k}").mat()
            assert np.array_equal(np.asarray(a).ravel(), want.ravel()), (side, k)
    assert got["size"] == (int(fs.getNode("LEFT.width").real()), int(fs.getNode("LEFT.height").real())) == (752, 480)
    fs.release()
