"""The refined pose on the GPU (the Levenberg-Marquardt tail of k_pnp_finalize in csrc/pnp.cu) against cv2 at 1e-8, on
the families of tests/test_oracle_lm_refine.py, and through the batched, streaming and multi-sequence modes.

Inlier lists equal cv2's and RANSAC iteration counts the oracle's on every set.  Then, per family:
  A  driving-like sets: rvec, tvec and R within 1e-8 absolute of cv2 (dropping one inlier from the sums moves the pose by
     1.5e-6 or more on these sets; stopping one iteration early by up to 4e-8);
  B  far or narrow clusters, flat along some directions: the cost over the inliers within 1e-10 relative of a scipy
     float64 optimum, the parameters within 1e-6 max(1, |p|) of cv2;
  C  runs into the 20-iteration cap with many rejected steps: parameters within 1e-8 max(1, |p|) of cv2, cost within
     1e-9 relative of cv2's."""
import numpy as np
import pytest

from visual_odom_b200 import synth

pytestmark = pytest.mark.gpu

cv2 = pytest.importorskip("cv2")
import test_oracle_lm_refine as L  # noqa: E402
from test_gpu_path import reference_unit  # noqa: E402
from test_gpu_triangulate_edges import _reference_drive, _sky_drive  # noqa: E402

POSE_TOL = 1e-8


def _pose_dist(got, rv, tv):
    R = cv2.Rodrigues(rv)[0]
    return max(np.abs(got["rvec"] - rv).max(), np.abs(got["tvec"] - tv).max(), np.abs(got["R"] - R).max())


def check_set(ctx, family, name):
    """ctx.pnp_ransac on one set against cv2 and the oracle; returns the family's deviation measure."""
    X, x, t_prev = L.lm_set(family, name)
    got = ctx.pnp_ransac(X, x, L.K, tvec0=t_prev)
    ok, rv, tv, inl = L.cv2_ransac(family, name)
    assert ok and np.array_equal(got["inliers"], inl), f"{name}: inlier list differs from cv2"
    assert got["iters"] == L.oracle_ransac(family, name)["iters"], f"{name}: RANSAC iterations differ from the oracle"
    p = np.concatenate([got["rvec"], got["tvec"]])
    Xi, xi = X[inl], x[inl]
    if family == "A":
        d = _pose_dist(got, rv, tv)
        assert d <= POSE_TOL, (name, d)
        return d
    scale = max(1.0, np.abs(np.concatenate([rv, tv])).max())
    d = np.abs(p - np.concatenate([rv, tv])).max() / scale
    if family == "B":
        c_opt = min(L.optimum(family, name)[1], L.cost(np.concatenate([rv, tv]), Xi, xi))
        rel = (L.cost(p, Xi, xi) - c_opt) / c_opt
        assert rel <= 1e-10, (name, rel)
        assert d <= 1e-6, (name, d)
        return rel
    c_cv2 = L.cost(np.concatenate([rv, tv]), Xi, xi)
    rel = abs(L.cost(p, Xi, xi) - c_cv2) / c_cv2
    assert d <= POSE_TOL, (name, d)
    assert rel <= 1e-9, (name, rel)
    return d


@pytest.mark.parametrize("family", "ABC")
def test_refined_pose_matches_cv2(ctx, family):
    worst, at = 0.0, None
    for name in L.FAMILIES[family]:
        d = check_set(ctx, family, name)
        if d >= worst:
            worst, at = d, name
    what = {"A": "|d(rvec, tvec, R)|", "B": "relative cost above the optimum", "C": "|dp| / max(1, |p|)"}[family]
    print(f"family {family}: worst {what} vs cv2 = {worst:.2e} ({at})")


# ----------------------------------------------------------------------------- the batched and sequence modes
def _check_record(got, R, t, where):
    d = max(np.abs(got["R"] - R).max(), np.abs(got["tvec"] - np.asarray(t).ravel()).max())
    assert d <= POSE_TOL, (where, d)
    return d


def test_frame_batch_units_of_different_sizes_in_both_orders(ctx):
    """vo_frame_batch with units of ~20 to ~2000 inliers in one launch, then in reversed order: every unit's R and t within
    1e-8 of the cv2 reference path, and identical in both orders."""
    w, h = 1241, 376
    t_prev = np.array([0.0, 0.0, -0.8])
    units = [(synth.stereo_unit(w, h, s, sky=sky), n) for s, n, sky in ((0, 2000, 0.0), (1, 60, 0.0), (2, 600, 0.35))]
    refs = [reference_unit(u, n, t_prev) for u, n in units]
    counts = sorted(len(r["inliers"]) for r in refs)
    assert counts[0] < 64 and counts[-1] > 1000, counts
    out = {}
    worst = 0.0
    for order in ([0, 1, 2], [2, 1, 0]):
        ctx.batch_configure(w, h, len(order), units[0][0]["P_l"], units[0][0]["P_r"])
        arr, keep, pitch = ctx.make_units([dict(units[i][0], n_select=units[i][1], t_prev=tuple(t_prev)) for i in order])
        res = ctx.frame_batch(arr, pitch)
        for k, i in enumerate(order):
            assert res[k]["n_inliers"] == len(refs[i]["inliers"]), (order, i)
            worst = max(worst, _check_record(res[k], refs[i]["R"], refs[i]["t"], f"unit {i} order {order}"))
            if i in out:
                assert np.array_equal(out[i]["R"], res[k]["R"]) and np.array_equal(out[i]["tvec"], res[k]["tvec"]), i
            out[i] = res[k]
    print(f"vo_frame_batch: worst |d[R|t]| vs cv2 = {worst:.2e}, inliers {counts}")


def test_sequence_modes_match_cv2(ctx):
    """A sky drive (zero-disparity band) and a dense drive through vo_seq_push and, together, through vo_mseq: every
    record's R and t within 1e-8 of the cv2 reference path."""
    drives = [_sky_drive(1241, 376, 31, synth.SEQ_STEP_R, synth.SEQ_STEP_T),
              _sky_drive(1241, 376, 7, (-0.002, 0.003, 0.0), (0.0, 0.0, -0.25), sky=0.0)]
    P_l, P_r = drives[0][0], drives[0][1]
    frames = [d[2] for d in drives]
    refs = [_reference_drive(P_l, P_r, fr) for fr in frames]
    worst = 0.0
    for q, fr in enumerate(frames):
        ctx.seq_begin(fr[0][0], fr[0][1], P_l, P_r)
        for k in range(1, len(fr)):
            got = ctx.seq_push(*fr[k])
            assert got["n_inliers"] == refs[q][k - 1]["n_inliers"], (q, k)
            worst = max(worst, _check_record(got, refs[q][k - 1]["R"], refs[q][k - 1]["t"], f"seq {q} frame {k}"))
    ctx.mseq_begin([fr[0][0] for fr in frames], [fr[0][1] for fr in frames], P_l, P_r)
    for k in range(1, len(frames[0])):
        ctx.mseq_submit([fr[k][0] for fr in frames], [fr[k][1] for fr in frames])
        recs = ctx.mseq_wait()
        for q in range(len(frames)):
            assert recs[q]["n_inliers"] == refs[q][k - 1]["n_inliers"], (q, k)
            worst = max(worst, _check_record(recs[q], refs[q][k - 1]["R"], refs[q][k - 1]["t"], f"mseq {q} frame {k}"))
    print(f"vo_seq / vo_mseq: worst |d[R|t]| vs cv2 = {worst:.2e}")
