"""FAST on the GPU (vo_fast_detect, the batched selection and sequence mode) against the oracle, bit for bit, at the
edges where the detector kernels can go wrong.

oracle/fast_ref.c is pinned list-exact against cv2 on the same images by tests/test_oracle_fast.py, so equality with
the oracle here is equality with cv::FAST.  Covered:
  * every threshold in {0, 1, 7, 20, 100, 254, 255} with non-max suppression on and off, each on a fresh context;
  * widths 7, 8, 2047..2050 and 4100 (k_fast_nms_row stages a row in passes of 2048 pixels with a 1-pixel halo) and
    heights 7, 8, 1025 and 2100 (k_fast_scan scans the row counts in chunks of 1024 rows), 1x1 and 6x6 frames, and a
    pitched view with poison bytes past the width;
  * a caller buffer smaller than the list, dense frames at the non-max suppression bound, and thresholds outside
    [0, 255], which vo_create refuses;
  * k_select_stride at N = 1, 2, 7, M-1, M, M+1 and the context capacity, and on a frame without corners;
  * dense frames (more corners than w*h/8) through the batched path and sequence mode, against the cv2 reference path;
  * one LK call on a frame whose level-0 rows are wider than 2048 pixels.
"""
import ctypes as C

import numpy as np
import pytest

from test_gpu_lk import _border_points
from test_gpu_path import check_unit, reference_unit          # the whole-path oracle and its comparison, shared
from test_gpu_seq import _frames as sequence_frames
from test_oracle_fast import (IMAGE_NAMES, SET_H, SET_W, THRESHOLDS, binary_noise, dense_tile, image_set, nms_bound,
                              ring_atlas, tie_atlas, uniform_noise)
from visual_odom_b200 import synth

pytestmark = pytest.mark.gpu

T_PREV = (0.0, 0.0, -0.8)


def _context(**params):
    from visual_odom_b200.capi import Context
    return Context(0, max_features=8192, **params)


def _detect(c, img, cap=None):
    """vo_fast_detect with its return code: (rc, n_out, points written, responses written)."""
    from visual_odom_b200.capi import _p
    img = np.asarray(img)
    h, w = img.shape
    cap = max(w * h, 1) if cap is None else cap
    out = np.full((cap, 2), -1, np.float32)
    resp = np.full(cap, -1, np.float32)
    n = C.c_int(-1)
    rc = c.lib.vo_fast_detect(c.h, _p(img), w, h, img.strides[0], _p(out), _p(resp), cap, C.byref(n))
    m = min(n.value, cap)
    return rc, n.value, out[:m], resp[:m]


def _check(c, img, t=20, nms=True):
    from oracle import cref
    from visual_odom_b200.capi import VO_OK
    ref_xy, ref_resp = cref.fast_detect(np.ascontiguousarray(img), threshold=t, nms=bool(nms))
    rc, n, xy, resp = _detect(c, img)
    assert rc == VO_OK, c.lib.vo_last_error(c.h).decode()
    assert n == len(ref_xy)
    assert np.array_equal(xy, ref_xy)                # coordinates and raster order
    assert np.array_equal(resp, ref_resp)            # scores with non-max suppression, 0 without
    return n


@pytest.fixture(scope="module")
def ctxs(built):
    """One context per fast_nonmax value at the default threshold, shared by the geometry tests."""
    cs = {nms: _context(fast_nonmax=nms) for nms in (1, 0)}
    yield cs
    for c in cs.values():
        c.close()


# ---- parameters ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nms", [1, 0])
@pytest.mark.parametrize("t", THRESHOLDS)
def test_thresholds_and_nonmax(built, t, nms):
    c = _context(fast_threshold=t, fast_nonmax=nms)
    try:
        imgs = image_set(SET_H, SET_W, t)
        counts = {name: _check(c, imgs[name], t, nms) for name in IMAGE_NAMES}
    finally:
        c.close()
    if t < 255:
        assert counts["ring_atlas"] > 100 and counts["binary"] > 0
    else:
        assert not any(counts.values())


def test_out_of_range_thresholds_refused(built):
    from visual_odom_b200.capi import VO_E_INVALID, VoError
    for t in (-1, 256, 1000):
        with pytest.raises(VoError) as e:
            _context(fast_threshold=t)
        assert e.value.code == VO_E_INVALID and "fast_threshold" in str(e.value)


# ---- geometry --------------------------------------------------------------------------------------------------------
def _geometry_images(h, w):
    return dict(uniform=uniform_noise(h, w, seed=w + h), binary=binary_noise(h, w, seed=w * h), tile=dense_tile(h, w),
                ring_atlas=ring_atlas(h, w, 20), ties=tie_atlas(h, w))


@pytest.mark.parametrize("nms", [1, 0])
@pytest.mark.parametrize("w,h", [(7, 48), (8, 48), (2047, 48), (2048, 48), (2049, 48), (2050, 48), (4100, 48),
                                 (300, 7), (300, 8), (300, 1025), (300, 2100)])
def test_geometry(ctxs, w, h, nms):
    from oracle import cref
    imgs = _geometry_images(h, w)
    assert sum(_check(ctxs[nms], img, 20, nms) for img in imgs.values()) > 0
    if w == 4100:                                    # the third NMS pass has corners to keep (x = 4096 is the last column)
        assert any((cref.fast_detect(img, nms=bool(nms))[0][:, 0] == 4096).any() for img in imgs.values())


@pytest.mark.parametrize("nms", [1, 0])
@pytest.mark.parametrize("w,h", [(1, 1), (6, 6), (6, 40), (40, 6)])
def test_frames_without_interior(ctxs, w, h, nms):
    from visual_odom_b200.capi import VO_OK
    rc, n, _, _ = _detect(ctxs[nms], uniform_noise(h, w))
    assert rc == VO_OK and n == 0


def test_pitched_view_with_poison(ctxs):
    h, w, pad = 200, 333, 35
    buf = binary_noise(h, w + pad, seed=11)          # bytes past the width: a kernel that reads them finds corners
    buf[:, :w] = uniform_noise(h, w, seed=12)
    view = buf[:, :w]
    assert view.strides[0] == w + pad
    for nms in (1, 0):
        assert _check(ctxs[nms], view, 20, nms) > 0


# ---- capacity --------------------------------------------------------------------------------------------------------
def test_caller_buffer_smaller_than_list(ctxs):
    from oracle import cref
    from visual_odom_b200.capi import VO_E_CAPACITY
    img = uniform_noise(SET_H, SET_W, seed=21)
    ref_xy, ref_resp = cref.fast_detect(img)
    for cap in (1, len(ref_xy) // 3, len(ref_xy) - 1):
        rc, n, xy, resp = _detect(ctxs[1], img, cap)
        assert rc == VO_E_CAPACITY and n == len(ref_xy)
        assert np.array_equal(xy, ref_xy[:cap]) and np.array_equal(resp, ref_resp[:cap])


@pytest.mark.parametrize("w,h", [(1241, 376), (1920, 1080)])
def test_dense_tile_whole_list(ctxs, w, h):
    n = _check(ctxs[1], dense_tile(h, w))
    assert n > max(w * h // 8, 65536) and n <= nms_bound(h, w)


# ---- selection and dense frames through the batched path -------------------------------------------------------------
def test_select_stride_edges(built):
    from oracle import cref
    from visual_odom_b200.capi import VO_E_TOO_FEW_POINTS
    w, h = 640, 240
    u = synth.stereo_unit(w, h, 3)
    corners, _ = cref.fast_detect(u["l0"])
    M = len(corners)
    c = _context()
    try:
        cap = c.params.max_features
        assert 8 < M < cap
        flat = np.full((h, w), 128, np.uint8)
        counts = [1, 2, 7, M - 1, M, M + 1, cap]
        units = [dict(u, n_select=n, t_prev=T_PREV) for n in counts]
        units.append(dict(l0=flat, r0=flat, l1=flat, r1=flat, P_l=u["P_l"], P_r=u["P_r"], n_select=2000, t_prev=T_PREV))
        c.batch_configure(w, h, len(units), u["P_l"], u["P_r"])
        arr, keep, pitch = c.make_units(units)
        res = c.frame_batch(arr, pitch)
        refs = {}
        for i, (unit, r) in enumerate(zip(units, res)):
            m = M if i < len(counts) else 0
            want = synth.select_features(corners if m else corners[:0], unit["n_select"])
            got = c.batch_fetch(i, r)
            assert r["n_detected"] == m and r["n_features"] == min(unit["n_select"], m) == len(want), i
            assert np.array_equal(got["pts_in"], want), i
            if r["n_valid"] < 4:
                assert r["pnp_status"] == VO_E_TOO_FEW_POINTS, i
            if i >= 3 and m:                              # M-1, M, M+1 and the capacity: the whole path against cv2
                key = min(unit["n_select"], M)
                if key not in refs:
                    refs[key] = reference_unit(u, unit["n_select"], np.array(T_PREV))
                check_unit(r, got, refs[key])
        assert res[0]["n_valid"] < 4 and res[1]["n_valid"] < 4 and res[-1]["n_valid"] == 0
    finally:
        c.close()


def _tile_band(img, rows=240):
    """The tile in the bottom `rows` rows.  The band is at the bottom because the features that survive the circular
    check come from the textured rows, and the far plane at the top of the synthetic scene tracks best: with the band
    at the top, fewer than 4 features of a 2000 survive and the reference path cannot solve a pose."""
    out = img.copy()
    out[-rows:] = dense_tile(rows, img.shape[1])
    return out


def test_dense_units_batched_vs_cv2(built):
    """Two KITTI-size units whose left image holds the tile in 240 of its rows: more corners than the old capacity of
    max(w*h/8, 65536), so the even-stride selection must run over the whole list."""
    pytest.importorskip("cv2")
    from oracle import cref
    w, h, n_sel = 1241, 376, 2000
    units = []
    for seed in (70, 71):
        u = synth.stereo_unit(w, h, seed, cal=synth.KITTI00)
        u["l0"] = _tile_band(u["l0"])
        assert len(cref.fast_detect(u["l0"])[0]) > max(w * h // 8, 65536)
        units.append(u)
    c = _context()
    try:
        c.batch_configure(w, h, len(units), units[0]["P_l"], units[0]["P_r"])
        arr, keep, pitch = c.make_units([dict(u, n_select=n_sel, t_prev=T_PREV) for u in units])
        res = c.frame_batch(arr, pitch)
        for i, u in enumerate(units):
            check_unit(res[i], c.batch_fetch(i, res[i]), reference_unit(u, n_sel, np.array(T_PREV)))
    finally:
        c.close()


def test_dense_full_hd_selection(built):
    from oracle import cref
    w, h, n_sel = 1920, 1080, 2000
    u = synth.stereo_unit(w, h, 72, cal=synth.ZED, scene="v0")
    u["l0"] = dense_tile(h, w)
    corners, _ = cref.fast_detect(u["l0"])
    assert len(corners) == nms_bound(h, w)
    c = _context()
    try:
        c.batch_configure(w, h, 1, u["P_l"], u["P_r"])
        arr, keep, pitch = c.make_units([dict(u, n_select=n_sel, t_prev=T_PREV)])
        r = c.frame_batch(arr, pitch)[0]
        assert r["n_detected"] == len(corners) and r["n_features"] == n_sel
        assert np.array_equal(c.batch_fetch(0, r)["pts_in"], synth.select_features(corners, n_sel))
    finally:
        c.close()


# ---- sequence mode on a dense frame ----------------------------------------------------------------------------------
def test_sequence_dense_frames_match_reference(built):
    """seq_begin on a frame whose left image holds the tile band, then two pushes: every refill appends more than the old
    capacity of corners.  Compared with the reference glue as test_gpu_seq.py does."""
    pytest.importorskip("cv2")
    from oracle import ref_path
    base, frames = sequence_frames(1241, 376, 33, 3)
    frames = [(_tile_band(l), r) for l, r in frames]
    c = _context()
    try:
        c.seq_begin(frames[0][0], frames[0][1], base["P_l"], base["P_r"])
        fs = ref_path.FeatureSet()
        translation = np.zeros(3)
        for k in range(1, len(frames)):
            l0, r0 = frames[k - 1]; l1, r1 = frames[k]
            got = c.seq_push(l1, r1)
            pL0, pR0, pL1, pR1, info = ref_path.matching_features(l0, r0, l1, r1, fs, backend="cv2")
            X = ref_path.triangulate(base["P_l"], base["P_r"], pL0, pR0, "cv2")
            R, translation, inl, rvec = ref_path.tracking_frame2frame(base["P_l"], pL0, pL1, X, translation, "cv2")
            assert got["n_detected"] > max(1241 * 376 // 8, 65536), f"frame {k}: the refill is not dense"
            assert got["n_features"] == len(info["bucketed"]), f"frame {k}: bucketed feature count"
            assert got["n_tracked"] == len(info["kept_idx"]) and got["n_valid"] == len(pL0)
            for name, ref in (("l0", pL0), ("r0", pR0), ("l1", pL1), ("r1", pR1)):
                assert np.array_equal(got[name], ref), f"frame {k}: {name}"
            assert got["n_inliers"] == len(inl), f"frame {k}: inlier count"
            assert np.linalg.norm(got["R"] - R) / np.linalg.norm(R) <= 1e-4
            assert np.linalg.norm(got["tvec"] - translation) / np.linalg.norm(translation) <= 1e-4
            pts, ages, t = c.seq_state()
            assert np.array_equal(pts, fs.points) and np.array_equal(ages, fs.ages), f"frame {k}: carried FeatureSet"
    finally:
        c.close()


# ---- pyramids and LK on rows wider than 2048 pixels ------------------------------------------------------------------
def test_lk_wide_rows(ctx):
    from oracle import cref
    w, h = 2600, 300
    u = synth.stereo_unit(w, h, 4, scene="v0")
    corners, _ = cref.fast_detect(u["l0"])
    pts = synth.select_features(corners, 4000)
    rng = np.random.default_rng(4)
    pts = np.concatenate([pts + rng.uniform(-0.5, 0.5, pts.shape).astype(np.float32), _border_points(w, h)])
    assert (pts[:, 0] > 2100).sum() > 500
    ro, rs, re = cref.lk_track(u["l0"], u["l1"], pts)
    go, gs, ge = ctx.lk_track(u["l0"], u["l1"], pts)
    assert np.array_equal(gs, rs), f"status differs at {np.nonzero(gs != rs)[0][:10]}"
    assert np.array_equal(go, ro), f"positions differ at {np.nonzero((go != ro).any(1))[0][:10]}"
    ok = rs == 1
    assert np.array_equal(ge[ok], re[ok]) and ok.sum() > 0.8 * len(pts)
