"""Triangulation on the GPU at zero and vanishing disparity, where cv::convertPointsFromHomogeneous stops dividing by w
(|w| <= FLT_EPSILON): the kernel on the disparity families of tests/test_oracle_triangulate_edges.py, and a far-field
scene (synth's `sky` band at infinity: identical left / right pixels, a rotation-only warp between times) through the
batched path, the streaming sequence mode and several sequences at once, each against cv2 through the reference's glue
(oracle/ref_path.py).  On such a scene LK returns its start position bit for bit on identical windows, so hundreds of
survivors have r0 == l0 exactly; cv2 keeps them as unit-norm columns within 1 m of the camera (PnP outliers), where
dividing by the DLT's w ~ 1e-18 would put them 1e17 m away, reprojecting along the pure rotation as inliers."""
import numpy as np
import pytest

import test_oracle_triangulate_edges as E  # noqa: E402
from test_gpu_path import check_unit, reference_unit  # noqa: E402
from visual_odom_b200 import synth

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")

SKY = 0.35
NF = 8


@pytest.mark.parametrize("cal", sorted(E.CALS))
@pytest.mark.parametrize("name", E.FAMILIES)
def test_kernel_bit_exact_with_cv2_on_edge_families(ctx, name, cal):
    P_l, P_r = synth.proj_matrices(E.CALS[cal][0])
    a, b = E.points(name, cal)
    H, X = E.cv2_triangulate(P_l, P_r, a, b)
    got = ctx.triangulate(P_l, P_r, a, b)
    got4 = ctx.triangulate_homogeneous(P_l, P_r, a, b)
    assert np.array_equal(got4, H), "homogeneous column"
    assert np.array_equal(got, X), "3-D point"
    E._edge_asserts(name, H, X)


@pytest.mark.parametrize("n", [1, 127, 128, 129, 255, 256, 257, 8191, 8192])
def test_kernel_point_counts_around_block_size_and_capacity(ctx, n):
    """Every family mixed and shuffled, n points: around k_triangulate's 128-thread blocks and at the context's 8192."""
    P_l, P_r = synth.proj_matrices(synth.KITTI00)
    parts = [E.points(name, "kitti") for name in E.FAMILIES]
    a = np.concatenate([p[0] for p in parts]); b = np.concatenate([p[1] for p in parts])
    idx = np.random.default_rng(n).permutation(np.resize(np.arange(len(a)), max(n, len(a))))[:n]
    a, b = E._f32(a[idx]), E._f32(b[idx])
    H, X = E.cv2_triangulate(P_l, P_r, a, b)
    assert np.array_equal(ctx.triangulate_homogeneous(P_l, P_r, a, b), H)
    assert np.array_equal(ctx.triangulate(P_l, P_r, a, b), X)
    if n >= 128:
        assert (np.abs(H[:, 3]) <= E.EPS).sum() > 0 and (np.abs(H[:, 3]) > E.EPS).sum() > 0


def _far_field(P_l, P_r, l0, r0):
    """(survivors with r0.x == l0.x exactly, points whose cv2 w has |w| <= FLT_EPSILON)."""
    if len(l0) == 0:
        return 0, 0
    w = np.abs(cv2.triangulatePoints(P_l, P_r, l0.T.copy(), r0.T.copy())[3])
    return int((r0[:, 0] == l0[:, 0]).sum()), int((w <= E.EPS).sum())


def _sky_drive(w, h, seed, step_r, step_t, n=NF, sky=SKY):
    base = synth.stereo_unit(w, h, seed, sky=sky)
    out = [(base["l0"], base["r0"])]
    for k in range(1, n):
        u = synth.stereo_unit(w, h, seed, rvec=np.asarray(step_r) * k, tvec=np.asarray(step_t) * k, sky=sky)
        out.append((u["l1"], u["r1"]))
    return base["P_l"], base["P_r"], out


@pytest.mark.parametrize("w,h,n_sel,cal", [(1241, 376, 2000, "kitti"), (1920, 1080, 4000, "zed")])
def test_far_field_batched_path_matches_cv2(ctx, w, h, n_sel, cal):
    c = synth.KITTI00 if cal == "kitti" else synth.ZED
    seeds = [0, 1] if cal == "kitti" else [2]
    units = [synth.stereo_unit(w, h, s, cal=c, sky=SKY) for s in seeds]
    t_prev = (0.0, 0.0, -0.8)
    ctx.batch_configure(w, h, len(units), units[0]["P_l"], units[0]["P_r"])
    arr, keep, pitch = ctx.make_units([dict(u, n_select=n_sel, t_prev=t_prev) for u in units])
    res = ctx.frame_batch(arr, pitch)
    for i, u in enumerate(units):
        ref = reference_unit(u, n_sel, np.array(t_prev))
        exact, tiny_w = _far_field(u["P_l"], u["P_r"], ref["l0"], ref["r0"])
        assert exact >= 100 and tiny_w >= 1, (exact, tiny_w)
        check_unit(res[i], ctx.batch_fetch(i, res[i]), ref)


def _reference_drive(P_l, P_r, frames):
    """Per frame: the reference's point lists, inlier count, R, translation and frame_pose (cv2 through the glue)."""
    from oracle import ref_path
    fs = ref_path.FeatureSet()
    translation = np.zeros(3)
    frame_pose = np.eye(4)
    out = []
    for k in range(1, len(frames)):
        (l0, r0), (l1, r1) = frames[k - 1], frames[k]
        pL0, pR0, pL1, pR1, info = ref_path.matching_features(l0, r0, l1, r1, fs, backend="cv2")
        X = ref_path.triangulate(P_l, P_r, pL0, pR0, "cv2")
        R, translation, inl, _ = ref_path.tracking_frame2frame(P_l, pL0, pL1, X, translation, "cv2")
        frame_pose = ref_path.integrate_pose(frame_pose, R, translation)
        out.append(dict(n_features=len(info["bucketed"]), l0=pL0, r0=pR0, l1=pL1, r1=pR1, n_inliers=len(inl), R=R,
                        t=translation.copy(), pose=frame_pose.copy(), points=fs.points.copy(), ages=fs.ages.copy()))
    return out


def _check_frame(got, pose, state, ref, where):
    assert got["n_features"] == ref["n_features"], f"{where}: bucketed feature count"
    for name in ("l0", "r0", "l1", "r1"):
        assert np.array_equal(got[name], ref[name]), f"{where}: {name}"
    assert got["n_inliers"] == ref["n_inliers"], f"{where}: inlier count"
    assert np.linalg.norm(got["R"] - ref["R"]) / np.linalg.norm(ref["R"]) <= 1e-4, f"{where}: R"
    assert np.linalg.norm(got["tvec"] - ref["t"]) / np.linalg.norm(ref["t"]) <= 1e-4, f"{where}: t"
    assert np.abs(pose - ref["pose"]).max() <= 1e-6 * max(1.0, np.abs(ref["pose"]).max()), f"{where}: frame_pose"
    pts, ages, _ = state
    assert np.array_equal(pts, ref["points"]) and np.array_equal(ages, ref["ages"]), f"{where}: carried FeatureSet"


def test_far_field_sequence_matches_cv2(ctx):
    P_l, P_r, frames = _sky_drive(1241, 376, 31, synth.SEQ_STEP_R, synth.SEQ_STEP_T)
    ref = _reference_drive(P_l, P_r, frames)
    ctx.seq_begin(frames[0][0], frames[0][1], P_l, P_r)
    exact = 0
    for k in range(1, NF):
        got = ctx.seq_push(*frames[k])
        _check_frame(got, ctx.seq_pose(), ctx.seq_state(), ref[k - 1], f"frame {k}")
        e, tiny_w = _far_field(P_l, P_r, ref[k - 1]["l0"], ref[k - 1]["r0"])
        assert tiny_w >= 1, f"frame {k}: no point at |w| <= FLT_EPSILON"
        exact += e
    assert exact >= 100
    assert np.linalg.norm(ctx.seq_pose()[:3, 3]) > 0.5 * (NF - 1) * np.linalg.norm(synth.SEQ_STEP_T)


def test_far_field_among_several_sequences_matches_cv2(ctx):
    """vo_mseq_*: two sky drives and one without the band, one launch per stage for all three, each against cv2."""
    drives = [_sky_drive(1241, 376, 31, synth.SEQ_STEP_R, synth.SEQ_STEP_T),
              _sky_drive(1241, 376, 7, (-0.002, 0.003, 0.0), (0.0, 0.0, -0.25), sky=0.0),
              _sky_drive(1241, 376, 13, (0.0, 0.002, -0.001), (-0.02, 0.004, -0.15))]
    P_l, P_r = drives[0][0], drives[0][1]
    frames = [d[2] for d in drives]
    refs = [_reference_drive(P_l, P_r, fr) for fr in frames]
    n = len(frames)
    ctx.mseq_begin([fr[0][0] for fr in frames], [fr[0][1] for fr in frames], P_l, P_r)
    exact = [0] * n
    for k in range(1, NF):
        ctx.mseq_submit([fr[k][0] for fr in frames], [fr[k][1] for fr in frames])
        recs = ctx.mseq_wait()
        for q in range(n):
            _check_frame(recs[q], ctx.mseq_pose(q), ctx.mseq_state(q), refs[q][k - 1], f"sequence {q} frame {k}")
            e, tiny_w = _far_field(P_l, P_r, refs[q][k - 1]["l0"], refs[q][k - 1]["r0"])
            exact[q] += e
            if q != 1:
                assert tiny_w >= 1, f"sequence {q} frame {k}: no point at |w| <= FLT_EPSILON"
    assert exact[0] >= 100 and exact[2] >= 100, exact
