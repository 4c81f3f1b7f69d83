"""k_lk_ring at the edges of calcOpticalFlowPyrLK, bit for bit against the oracle (oracle/lk_ref.c) and against cv2 where
it is importable: the mined edge fixture (tests/golden/lk_edges/lk_edges.npz) under every LK launch configuration, window-bound
starts in closed form, every pyramid-depth transition and images smaller than the window, saturated images, and host
images whose row pitch is not their width."""
import json
import os
import sys

import numpy as np
import pytest

from visual_odom_b200 import synth

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_lk_edges as mk          # noqa: E402

SPANS = (0, 1, 2, 3, 5, 7, 16)      # tests/test_gpu_lk_variants.py
CONFIGS = [dict()] + [dict(lk_span=s) for s in SPANS] + [dict(lk_staging=1, lk_span=s) for s in SPANS]


def _cv2():
    try:
        import cv2
        return cv2
    except ImportError:
        return None


def _single_refs(a, b, pts):
    """(oracle, cv2 or None) results of one call"""
    from oracle import cref
    ref = cref.lk_track(a, b, pts)
    cv2 = _cv2()
    if cv2 is None:
        return ref, None
    crit = (cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, 30, 0.01)
    o, s, e = cv2.calcOpticalFlowPyrLK(a, b, np.ascontiguousarray(pts, np.float32).reshape(-1, 1, 2), None,
                                       winSize=(21, 21), maxLevel=3, criteria=crit, flags=0, minEigThreshold=0.001)
    return ref, (o.reshape(-1, 2), s.ravel(), e.ravel())


def _assert_single(got, ref, what):
    go, gs, ge = got
    ro, rs, re = ref
    assert np.array_equal(gs, rs), f"{what}: status differs at {np.nonzero(gs != rs)[0][:8]}"
    bad = np.nonzero((go != ro).any(1))[0]
    assert len(bad) == 0, f"{what}: positions differ at {len(bad)} points, first {bad[:8]}"
    assert np.array_equal(ge[rs == 1], re[rs == 1]), what


def _check_single(ctx, a, b, pts, what):
    ref, cvr = _single_refs(a, b, pts)
    got = ctx.lk_track(a, b, pts)
    _assert_single(got, ref, f"{what} vs oracle")
    if cvr is not None:
        _assert_single(got, cvr, f"{what} vs cv2")
    return ref


def _check_ring(ctx, imgs, pts, what):
    from oracle import ref_path
    fs = ref_path.FeatureSet()
    fs.points = pts.copy(); fs.ages = np.arange(len(pts), dtype=np.int32) % 5
    ages0 = fs.ages.copy()
    ref = ref_path.circular_matching(*imgs, pts, fs, backend="c")
    got = ctx.circular_match(*imgs, pts, ages=ages0)
    assert np.array_equal(got["status4"], ref["raw"]["status"]), f"{what}: ring status differs"
    for k, name in enumerate(("r0", "r1", "l1", "l0_ret")):
        bad = np.nonzero((got["raw4"][k] != ref["raw"][name]).any(1))[0]
        assert len(bad) == 0, f"{what}: call {k} differs at {len(bad)} points, first {bad[:8]}"
    assert np.array_equal(got["kept_idx"], ref["kept_idx"]), what
    assert np.array_equal(got["ages"], fs.ages), what
    if _cv2() is not None:
        cvr = ref_path.circular_matching(*imgs, pts, ref_path.FeatureSet(), backend="cv2")["raw"]
        assert np.array_equal(cvr["status"], ref["raw"]["status"]), f"{what}: oracle ring status differs from cv2"
        for name in ("r0", "r1", "l1", "l0_ret"):
            assert np.array_equal(cvr[name], ref["raw"][name]), f"{what}: oracle ring differs from cv2 ({name})"
    return ref


# ---- the mined fixture under every launch configuration --------------------------------------------------------------
@pytest.fixture(scope="module")
def edges(built):
    fx = np.load(os.path.join(HERE, "golden", "lk_edges", "lk_edges.npz"))
    out = []
    for ri, r in enumerate(json.loads(str(fx["recipes"]))):
        imgs = mk.images(r)
        assert [mk.sha(a) for a in imgs] == json.loads(str(fx[f"sha256_{ri}"]))
        out.append(dict(imgs=imgs, pts=fx[f"pts_{ri}"], out=fx[f"out_{ri}"], status=fx[f"status_{ri}"],
                        err=fx[f"err_{ri}"]))
    return out


@pytest.mark.parametrize("i", range(len(CONFIGS)),
                         ids=["default"] + ["-".join(f"{k}={v}" for k, v in c.items()) for c in CONFIGS[1:]])
def test_edge_fixture_bit_exact(edges, i):
    """The fixture's points (stored outputs = cv2 = oracle): call L0 -> R0 through vo_lk_track, the ring through
    vo_circular_match, on a fresh context per configuration."""
    from visual_odom_b200.capi import Context
    c = Context(0, max_features=8192)
    try:
        for k, v in CONFIGS[i].items():
            c.set_option(k, v)
        for ri, e in enumerate(edges):
            imgs, pts = e["imgs"], e["pts"]
            go, gs, ge = c.lk_track(imgs[0], imgs[1], pts)
            _assert_single((go, gs, ge), (e["out"][0], e["status"][0], e["err"][0]), f"recipe {ri} single call")
            got = c.circular_match(*imgs, pts)
            assert np.array_equal(got["status4"], e["status"]), f"recipe {ri}: ring status"
            for k in range(4):
                bad = np.nonzero((got["raw4"][k] != e["out"][k]).any(1))[0]
                assert len(bad) == 0, f"recipe {ri}: ring call {k} differs at {bad[:8]}"
    finally:
        c.close()


# ---- the convergence test decided in double ------------------------------------------------------------------------
ITER_KINDS = (0, 1, 2, 3)           # oracle/cref.py EV_ITER, EV_EPS, EV_HALF, EV_CAP


def _eps_flip_cases(a, b, pts, want):
    """(start, epsilon) pairs whose track, at that epsilon, has an iteration where delta.ddot(delta) <= eps^2 (double, as
    OpenCV decides) and the float-only test (float)(dx^2 + dy^2) <= (float)eps^2 disagree.  At eps = 0.01 such an
    iteration is rarer than one in 10^8; choosing eps from a logged step makes one per start.  One case per start."""
    from oracle import cref
    _, _, _, log = cref.lk_track(a, b, pts, return_log=True)
    it = log[np.isin(log["kind"], ITER_KINDS) & (log["d2"] > 1e-6) & (log["d2"] < 1e-2)]
    out, used = [], set()
    for ev in it:
        if int(ev["pt"]) in used:
            continue
        d2, d2f = float(ev["d2"]), ev["d2f"]
        target = d2 if np.float32(d2) < d2f else np.nextafter(d2, 0)
        for eps in (np.sqrt(target), np.nextafter(np.sqrt(target), 1), np.nextafter(np.sqrt(target), 0)):
            e2 = eps * eps
            if (d2 <= e2) != (d2f <= np.float32(e2)):
                break
        else:
            continue
        p = pts[ev["pt"]][None]
        lg = cref.lk_track(a, b, p, epsilon=float(eps), return_log=True)[3]
        li = lg[np.isin(lg["kind"], ITER_KINDS)]
        if ((li["d2"] <= e2) != (li["d2f"] <= np.float32(e2))).any():
            out.append((p, float(eps)))
            used.add(int(ev["pt"]))
            if len(out) == want:
                break
    return out


def test_eps_decided_in_double(built):
    """Contexts whose lk_epsilon puts an iteration between the double and the float form of the convergence test."""
    from oracle import cref
    from visual_odom_b200.capi import Context
    u = synth.stereo_unit(1241, 376, 5)
    corners, _ = cref.fast_detect(u["l0"])
    cases = _eps_flip_cases(u["l0"], u["r0"], synth.select_features(corners, 600), 8)
    assert len(cases) == 8
    cv2 = _cv2()
    for p, eps in cases:
        c = Context(0, max_features=64, lk_epsilon=eps)
        try:
            got = c.lk_track(u["l0"], u["r0"], p)
        finally:
            c.close()
        _assert_single(got, cref.lk_track(u["l0"], u["r0"], p, epsilon=eps), f"eps {eps!r} at {p[0]}")
        if cv2 is not None:
            crit = (cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, 30, eps)
            o, s, e = cv2.calcOpticalFlowPyrLK(u["l0"], u["r0"], p.reshape(-1, 1, 2), None, winSize=(21, 21), maxLevel=3,
                                               criteria=crit, flags=0, minEigThreshold=0.001)
            _assert_single(got, (o.reshape(-1, 2), s.ravel(), e.ravel()), f"eps {eps!r} at {p[0]} vs cv2")


# ---- window-bound starts in closed form ----------------------------------------------------------------------------
def _bound_starts(w, h, nlev):
    """At level l the I window's origin floor(x / 2^l - 10) is in range iff -11 * 2^l <= x < (lw + 10) * 2^l: both bounds
    and the float just below each, for every level, in x (y mid-image) and in y (x mid-image)."""
    lw, lh = w, h
    sizes = []
    for l in range(nlev):
        sizes.append((lw, lh))
        lw, lh = (lw + 1) // 2, (lh + 1) // 2
    pts = []
    for l, (lw, lh) in enumerate(sizes):
        s = float(1 << l)
        for lo, hi, mid, axis in ((-11 * s, (lw + 10) * s, h / 2 + 0.3, 0), (-11 * s, (lh + 10) * s, w / 2 + 0.3, 1)):
            for v in (lo, hi):
                for x in (np.float32(v), np.nextafter(np.float32(v), np.float32(-np.inf))):
                    pts.append((x, mid) if axis == 0 else (mid, x))
    return np.array(pts, np.float32)


def test_window_bound_starts(ctx):
    w, h = 1241, 376
    u = synth.stereo_unit(w, h, 31)
    imgs = [u[k] for k in ("l0", "r0", "l1", "r1")]
    pts = _bound_starts(w, h, 4)
    # a start outside level 0 still carries the estimate of the coarser levels into its (status 0) output position
    _check_single(ctx, imgs[0], imgs[1], pts, "window bounds")
    _check_ring(ctx, imgs, pts, "window bounds ring")


# ---- pyramid depth -------------------------------------------------------------------------------------------------
# (w, h, levels): each side of the sizes where the coarsest level is 22 px (42/43, 84/85, 168/169), in width and in height
# separately; a one-level image; images narrower / shorter than the window
SIZES = [(42, 300, 1), (43, 300, 2), (84, 300, 2), (85, 300, 3), (168, 300, 3), (169, 300, 4),
         (500, 42, 1), (500, 43, 2), (500, 84, 2), (500, 85, 3), (500, 168, 3), (500, 169, 4),
         (40, 30, 1), (20, 200, 1), (200, 20, 1), (7, 60, 1), (60, 5, 1), (3, 3, 1)]


@pytest.mark.parametrize("w,h,nlev", SIZES)
def test_pyramid_depth_and_tiny_images(ctx, w, h, nlev):
    from oracle import cref
    u = synth.stereo_unit(1241, 376, 41)
    imgs = [np.ascontiguousarray(u[k][100:100 + h, 300:300 + w]) for k in ("l0", "r0", "l1", "r1")]
    assert cref.Pyramid(imgs[0]).nlevels() == nlev
    rng = np.random.default_rng(w * 1000 + h)
    pts = np.concatenate([np.stack([rng.uniform(-25, w + 25, 300), rng.uniform(-25, h + 25, 300)], 1),
                          np.stack([rng.uniform(0, w, 200), rng.uniform(0, h, 200)], 1),
                          _bound_starts(w, h, nlev)]).astype(np.float32)
    _check_single(ctx, imgs[0], imgs[1], pts, f"{w}x{h}")
    _check_ring(ctx, imgs, pts, f"{w}x{h} ring")


# ---- saturated images ----------------------------------------------------------------------------------------------
def test_saturated_images(ctx):
    """Random 2x2 blocks of 0 / 255 against their inverse and against a shifted copy: the largest gradients (|Scharr| up
    to 16 * 255 = 4080) and residuals (32 * 255 = 8160).  The kernel's per-chain sums of |addend| are unsigned 32-bit;
    the oracle's log gives the largest they reach here."""
    from oracle import cref
    w, h = 1241, 376
    rng = np.random.default_rng(7)
    blocks = rng.integers(0, 2, ((h + 1) // 2, (w + 1) // 2)).astype(np.uint8) * 255
    a = np.ascontiguousarray(np.kron(blocks, np.ones((2, 2), np.uint8))[:h, :w])
    inv = 255 - a
    shifted = np.ascontiguousarray(np.roll(a, (1, 3), (0, 1)))
    pts = np.stack([rng.uniform(0, w, 5000), rng.uniform(0, h, 5000)], 1).astype(np.float32)
    worst = np.zeros(10, np.int64)
    for b in (inv, shifted):
        ref = _check_single(ctx, a, b, pts, "saturated")
        assert ref[1].sum() > 0
        log = cref.lk_track(a, b, pts, return_log=True)[3]
        worst = np.maximum(worst, log["sabs"].max(0))
        _check_ring(ctx, [a, b, inv if b is shifted else shifted, a], pts, "saturated ring")
    print(f"largest sum |addend| per chain (b1 x4, tail, b2 x4, tail): {worst.tolist()}; 2^32 = {1 << 32}")
    assert worst.max() < 1 << 32
    assert worst.max() > 1 << 24          # the exact integer fast path is not taken on these


# ---- host images whose pitch is not their width ----------------------------------------------------------------------
def test_row_pitch_not_width(ctx):
    w, h = 333, 129
    u = synth.stereo_unit(w, h, 13, scene="v0")
    imgs = []
    for k in ("l0", "r0", "l1", "r1"):
        wide = np.zeros((h, w + 45), np.uint8)
        wide[:, 7:7 + w] = u[k]
        imgs.append(wide[:, 7:7 + w])          # a view: row pitch w + 45, passed as the C-ABI pitch
    assert imgs[0].strides == (w + 45, 1) and not imgs[0].flags.c_contiguous
    from oracle import cref
    corners, _ = cref.fast_detect(u["l0"])
    pts = np.concatenate([synth.select_features(corners, 400), _bound_starts(w, h, 3)]).astype(np.float32)
    ref, _ = _single_refs(u["l0"], u["r0"], pts)
    _assert_single(ctx.lk_track(imgs[0], imgs[1], pts), ref, "pitched single call")
    _check_ring(ctx, imgs, pts, "pitched ring")


def test_status_without_err(ctx):
    """err not requested: positions and status are those of the call that requests it."""
    u = synth.stereo_unit(1241, 376, 31)
    pts = _bound_starts(1241, 376, 4)
    go, gs, _ = ctx.lk_track(u["l0"], u["r0"], pts)
    no, ns, ne = ctx.lk_track(u["l0"], u["r0"], pts, want_err=False)
    assert ne is None and np.array_equal(ns, gs) and np.array_equal(no, go)
