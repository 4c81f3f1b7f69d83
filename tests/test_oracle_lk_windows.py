"""The oracle's lk_track (oracle/lk_ref.c) at every square window from 3x3 to 32x32, bit for bit against cv2 4.13.0:
positions, status and err on blurred noise, a KITTI-size stereo pair with starts beyond the border and saturated 0 / 255
blocks; the pyramid depth, which stops once a level is not larger than the window; and the windowed reference glue of
lk_window_scenes.py, which at 21 x 21 is oracle/ref_path.py's."""
import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")
import lk_window_scenes as S  # noqa: E402


@pytest.fixture(scope="module")
def scenes(built):
    return {name: make() for name, make in S.SCENES.items()}


def _cv_lk(a, b, pts, win):
    crit = (cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, 30, 0.01)
    o, s, e = cv2.calcOpticalFlowPyrLK(a, b, pts.reshape(-1, 1, 2), None, winSize=(win, win), maxLevel=3, criteria=crit,
                                       flags=0, minEigThreshold=0.001)
    return o.reshape(-1, 2), s.ravel(), e.ravel()


@pytest.mark.parametrize("win", S.WINDOWS)
def test_lk_track_matches_cv2_at_every_window(scenes, win):
    from oracle import cref
    for name, (a, b, pts) in scenes.items():
        co, cs, ce = _cv_lk(a, b, pts, win)
        o, s, e = cref.lk_track(a, b, pts, win=win)
        assert np.array_equal(s, cs), f"{name} W={win}: status differs at {np.nonzero(s != cs)[0][:8]}"
        assert np.array_equal(o, co), f"{name} W={win}: positions differ at {np.nonzero((o != co).any(1))[0][:8]}"
        assert np.array_equal(e[cs == 1], ce[cs == 1]), f"{name} W={win}: err"
        assert 0 < cs.sum() < len(pts), f"{name} W={win}: both outcomes"


@pytest.mark.parametrize("shape,max_level,depths", [
    ((44, 100), 3, {3: 4, 5: 4, 10: 3, 11: 2, 21: 2, 22: 1, 32: 1}),
    ((376, 1241), 7, {3: 7, 21: 5, 32: 4}),
])
def test_pyramid_depth_depends_on_the_window(built, shape, max_level, depths):
    from oracle import cref
    img = np.random.default_rng(0).integers(0, 256, shape).astype(np.uint8)
    for win, n in depths.items():
        assert cref.Pyramid(img, win, max_level).nlevels() == n, (shape, win)
        _, pyr = cv2.buildOpticalFlowPyramid(img, (win, win), max_level, withDerivatives=False)
        assert len(pyr) == n, (shape, win)


@pytest.mark.parametrize("backend", ["c", "cv2"])
def test_windowed_glue_at_21_is_the_reference_glue(built, backend):
    from oracle import ref_path
    from visual_odom_b200 import synth
    u = synth.stereo_unit(640, 240, 3)
    v = synth.stereo_unit(640, 240, 3, rvec=synth.SEQ_STEP_R, tvec=synth.SEQ_STEP_T)
    frames = [(u["l0"], u["r0"]), (u["l1"], u["r1"]), (v["l1"], v["r1"])]
    fa, fb = ref_path.FeatureSet(), ref_path.FeatureSet()
    for k in range(1, len(frames)):
        args = frames[k - 1] + frames[k]
        ref = ref_path.matching_features(*args, fa, backend)
        got = S.matching_features(*args, fb, 21, backend)
        for r, g in zip(ref[:4], got[:4]):
            assert np.array_equal(r, g), k
        assert np.array_equal(ref[4]["kept_idx"], got[4]["kept_idx"]) and np.array_equal(ref[4]["bucketed"], got[4]["bucketed"])
        assert np.array_equal(fa.points, fb.points) and np.array_equal(fa.ages, fb.ages), k
        assert len(ref[0]) > 50
