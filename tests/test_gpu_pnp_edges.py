"""The PnP tail on the GPU (k_pnp_* in csrc/pnp.cu, the mono branch in csrc/ess.cu) at its edges, against cv2 and the
oracle, on the sets tests/test_oracle_pnp_edges.py builds and pins: the five-point case, the RANSAC wave edges, ties,
degenerate scenes, points on the inlier threshold, the compaction's chunk and capacity edges, and units with 2 .. 400
survivors in one batch.  The RANSAC iteration count is asserted equal to the oracle's everywhere."""
import numpy as np
import pytest

from visual_odom_b200 import synth

pytestmark = pytest.mark.gpu

cv2 = pytest.importorskip("cv2")
import test_oracle_pnp_edges as E  # noqa: E402
from visual_odom_b200.capi import VoError, VO_E_CAPACITY, VO_E_TOO_FEW_POINTS  # noqa: E402


def check_gpu(ctx, X, x, K, res, tol=1e-4, t_prev=E.T_PREV):
    """ctx.pnp_ransac against cv2 (inliers identical, [R|t] within tol) and the oracle (iterations identical)."""
    got = ctx.pnp_ransac(X, x, K, tvec0=t_prev)
    ok, rv, tv, inl = E.cv2_pnp(X, x, K, t_prev)
    assert np.array_equal(got["inliers"], inl), "inlier list differs from cv2"
    assert got["iters"] == res["iters"], (got["iters"], res["iters"])
    if not ok:                                             # VO_PNP_NO_MODEL: the caller's guess
        assert np.array_equal(got["R"], np.eye(3)) and np.array_equal(got["tvec"], t_prev) and got["iters"] == 500
        return got, 0.0
    R, _ = cv2.Rodrigues(rv)
    d = max(np.abs(got["R"] - R).max(), np.abs(got["tvec"] - tv).max())
    assert d <= tol, d
    return got, d


def test_five_points(ctx):
    """n == 5: one unrefined EPnP on all five, iterations 0, [R|t] within 1e-9 of cv2 (the same operations; only the device
    libm's rounding differs); five identical points keep cv2's finite components (rvec 0, R = I, tvec nan)."""
    worst = 0.0
    for X, x, K in E.five_point_sets():
        res = E.oracle_pnp(X, x, K)
        got, d = check_gpu(ctx, X, x, K, res, tol=1e-9)
        worst = max(worst, d)
    print(f"n == 5: worst |d[R|t]| vs cv2 = {worst:.2e}")
    X, x, K = E.identical_five()
    ok, rv, tv, inl = E.cv2_pnp(X, x, K)
    got = ctx.pnp_ransac(X, x, K, tvec0=E.T_PREV)
    assert np.array_equal(got["inliers"], np.arange(5)) and got["iters"] == 0
    for g, w in ((got["rvec"], rv), (got["tvec"], tv)):
        assert np.array_equal(np.isfinite(g), np.isfinite(w)) and np.array_equal(g[np.isfinite(w)], w[np.isfinite(w)])
    assert np.array_equal(got["R"], np.eye(3))


@pytest.mark.parametrize("name", sorted(E.WAVE_SPECS))
def test_wave_sets(ctx, name):
    X, x, K, res, r = E.wave_set(name)
    got, _ = check_gpu(ctx, X, x, K, res)
    assert got["iters"] == r["iters"]


@pytest.mark.parametrize("name", E.DEGENERATE)
def test_degenerate_sets(ctx, name):
    X, x, K, res = E.degenerate_set(name)
    check_gpu(ctx, X, x, K, res)


def test_threshold_boundary(ctx):
    """Points whose squared f32 error is 0.25f or one ulp either side: the kernels' unfused sum decides as cv2's does."""
    X, x, K, res, moved, want = E.threshold_set()
    got, _ = check_gpu(ctx, X, x, K, res)
    inl = set(got["inliers"].tolist())
    assert [i in inl for i in moved] == want.tolist()


@pytest.mark.parametrize("n,sigma,outl,seed", [(1500, 0.05, 0.1, 0), (1500, 0.15, 0.3, 1), (1500, 0.2, 0.5, 2),
                                              (1500, 0.25, 0.6, 3), (300, 0.1, 0.2, 4), (60, 0.3, 0.4, 5), (5, 0.0, 0.0, 6)])
def test_stress_cases_iteration_count(ctx, n, sigma, outl, seed):
    """The stress cases of test_gpu_stages.py: the iteration count equals the oracle's."""
    X, x, K = E._stress(n, sigma, outl, seed)
    check_gpu(ctx, X, x, K, E.oracle_pnp(X, x, K))


@pytest.mark.parametrize("n", [257, 4097, 8191, 8192])
def test_counts_across_compaction_chunks_and_capacity(ctx, n):
    """Several 256-point chunks of k_pnp_finalize's ordered compaction, and the context's max_features (8192)."""
    X, x, K = E._stress(n, 0.1, 0.2, n)
    check_gpu(ctx, X, x, K, E.oracle_pnp(X, x, K))


def test_over_capacity(ctx):
    X, x, K = E._stress(8193, 0.1, 0.2, 1)
    with pytest.raises(VoError) as e:
        ctx.pnp_ransac(X, x, K)
    assert e.value.code == VO_E_CAPACITY


# ----------------------------------------------------------------------------- small units through vo_frame_batch
def reference_given(u, pts, t_prev):
    """reference_unit of test_gpu_path.py without detection and selection: the given features go straight into
    circularMatching; None for the pose where cv2 would abort (fewer than 4 survivors)."""
    from oracle import ref_path
    fs = ref_path.FeatureSet(); fs.points = pts.copy(); fs.ages = np.zeros(len(pts), np.int32)
    cm = ref_path.circular_matching(u["l0"], u["r0"], u["l1"], u["r1"], pts, fs, "cv2")
    ok = ref_path.check_valid_match(cm["l0"], cm["l0_ret"], 0)
    pL0, pR0, pL1, pR1 = (ref_path.remove_invalid_points(cm[k], ok) for k in ("l0", "r0", "l1", "r1"))
    X = ref_path.triangulate(u["P_l"], u["P_r"], pL0, pR0, "cv2")
    ref = dict(n_detected=0, pts=pts, kept3=cm["kept_idx"], kept=cm["kept_idx"][ok], l0=pL0, r0=pR0, l1=pL1, r1=pR1, X=X,
               R=None, t=None, inliers=np.zeros(0, np.int32))
    if len(pL0) >= 4:
        ref["R"], ref["t"], ref["inliers"], _ = ref_path.tracking_frame2frame(u["P_l"], pL0, pL1, X, t_prev, "cv2")
    return ref


@pytest.fixture(scope="module")
def small_units():
    """Given-feature units with 2, 4, 5, 5, 6 and ~400 survivors of the circular check, chosen from the kept list of a
    reference run: tracking is per feature, so the same features survive again.  The second five-point unit is 4 RANSAC
    inliers and 1 non-inlier of that run."""
    from oracle import cref
    from test_gpu_path import reference_unit
    u = synth.stereo_unit(640, 240, 3)
    t_prev = np.array([0.0, 0.0, -0.8])
    full = reference_unit(u, 500, t_prev)
    pts, kept, inl = full["pts"], full["kept"], full["inliers"]
    outl = np.setdiff1d(np.arange(len(kept)), inl)
    sel = {"n2": kept[:2], "n4": kept[:4], "n5": kept[:5], "n5_outlier": np.sort(kept[np.r_[inl[:4], outl[:1]]]),
           "n6": kept[:6], "n400": kept[:400]}
    units = {k: pts[v] for k, v in sel.items()}
    assert len(cref.fast_detect(u["l0"])[0]) > 0 and len(outl) > 0
    return u, units, t_prev


def _run_batch(ctx, u, units, order, t_prev):
    ctx.batch_configure(640, 240, len(order), u["P_l"], u["P_r"])
    arr, keep, pitch = ctx.make_units([dict(u, pts=units[k], t_prev=tuple(t_prev)) for k in order])
    res = ctx.frame_batch(arr, pitch)
    return {k: (res[i], ctx.batch_fetch(i, res[i])) for i, k in enumerate(order)}


def test_small_units_in_one_batch(ctx, small_units):
    """n < 4 gets VO_E_TOO_FEW_POINTS (cv2 asserts); 4, 5 (also with an outlier), 6 and ~400 survivors match the reference
    path; none of this depends on the other units of the batch or their order."""
    from test_gpu_path import check_unit
    u, units, t_prev = small_units
    order = list(units)
    out = _run_batch(ctx, u, units, order, t_prev)
    for k in order:
        r, got = out[k]
        ref = reference_given(u, units[k], t_prev)
        assert r["n_valid"] == len(ref["l0"]), k
        if ref["R"] is None:
            assert r["n_valid"] < 4 and r["pnp_status"] == VO_E_TOO_FEW_POINTS, k
            continue
        check_unit(r, got, ref)
        if k.startswith("n5"):
            assert r["n_valid"] == 5 and r["ransac_iters"] == 0 and r["pnp_status"] == 0, k
    rev = _run_batch(ctx, u, units, order[::-1], t_prev)
    for k in order:
        (a, ga), (b, gb) = out[k], rev[k]
        assert a["pnp_status"] == b["pnp_status"] and a["ransac_iters"] == b["ransac_iters"], k
        assert np.array_equal(ga["inliers"], gb["inliers"]) and np.array_equal(a["tvec"], b["tvec"], equal_nan=True), k


# ----------------------------------------------------------------------------- mono branch
def test_mono_five_points(ctx):
    """n == 5: vo_mono_rotation refuses exactly where cv2's recoverPose raises, and agrees where it does not."""
    refused = single = 0
    for p0, p1, focal, pp in E.mono_five_sets():
        ref, ncand = E.cv2_mono_or_none(p0, p1, focal, pp)
        if ref is None:
            with pytest.raises(VoError) as e:
                ctx.mono_rotation(p0, p1, focal, pp)
            assert e.value.code == VO_E_TOO_FEW_POINTS
            refused += 1
            continue
        Rg, mg, iters = ctx.mono_rotation(p0, p1, focal, pp)
        assert np.all(mg) and iters == 0 and np.abs(Rg - ref[0]).max() <= 1e-6
        single += 1
    print(f"mono n == 5 on the GPU: {refused} refused, {single} agree")
    assert refused > 0
