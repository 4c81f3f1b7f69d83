"""k_lk_ring at the edges of calcOpticalFlowPyrLK, bit for bit against the oracle (oracle/lk_ref.c) and against cv2 where
it is importable: the mined edge fixture (tests/golden/lk_edges/lk_edges.npz) under every LK launch configuration, window-bound
starts in closed form, every pyramid-depth transition and images smaller than the window, saturated images, and host
images whose row pitch is not their width.  The helpers take the window; the pyramid-depth test also runs k_lk_win at one
or more windows of each of its classes (tests/test_gpu_lk_win_edges.py has the rest of k_lk_win's edges)."""
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
CONFIGS = [dict()] + [dict(lk_span=s) for s in SPANS]


def _cv2():
    try:
        import cv2
        return cv2
    except ImportError:
        return None


def _single_refs(a, b, pts, win=21):
    """(oracle, cv2 or None) results of one call"""
    from oracle import cref
    ref = cref.lk_track(a, b, pts, win=win)
    cv2 = _cv2()
    if cv2 is None:
        return ref, None
    crit = (cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, 30, 0.01)
    o, s, e = cv2.calcOpticalFlowPyrLK(a, b, np.ascontiguousarray(pts, np.float32).reshape(-1, 1, 2), None,
                                       winSize=(win, win), maxLevel=3, criteria=crit, flags=0, minEigThreshold=0.001)
    return ref, (o.reshape(-1, 2), s.ravel(), e.ravel())


def _assert_single(got, ref, what):
    go, gs, ge = got
    ro, rs, re = ref
    assert np.array_equal(gs, rs), f"{what}: status differs at {np.nonzero(gs != rs)[0][:8]}"
    bad = np.nonzero((go != ro).any(1))[0]
    assert len(bad) == 0, f"{what}: positions differ at {len(bad)} points, first {bad[:8]}"
    assert np.array_equal(ge[rs == 1], re[rs == 1]), what


def _check_single(ctx, a, b, pts, what, win=21):
    ref, cvr = _single_refs(a, b, pts, win)
    got = ctx.lk_track(a, b, pts)
    _assert_single(got, ref, f"{what} vs oracle")
    if cvr is not None:
        _assert_single(got, cvr, f"{what} vs cv2")
    return ref


def _circular(imgs, pts, fs, win, backend):
    """the reference's circularMatching on the oracle ("c") or on cv2, at a win x win window"""
    from oracle import ref_path
    if win == 21:
        return ref_path.circular_matching(*imgs, pts, fs, backend=backend)
    import lk_window_scenes as S
    return S.circular_matching(*imgs, pts, fs, win, backend)


def _check_ring(ctx, imgs, pts, what, win=21):
    from oracle import ref_path
    fs = ref_path.FeatureSet()
    fs.points = pts.copy(); fs.ages = np.arange(len(pts), dtype=np.int32) % 5
    ages0 = fs.ages.copy()
    ref = _circular(imgs, pts, fs, win, "c")
    got = ctx.circular_match(*imgs, pts, ages=ages0)
    assert np.array_equal(got["status4"], ref["raw"]["status"]), f"{what}: ring status differs"
    for k, name in enumerate(("r0", "r1", "l1", "l0_ret")):
        bad = np.nonzero((got["raw4"][k] != ref["raw"][name]).any(1))[0]
        assert len(bad) == 0, f"{what}: call {k} differs at {len(bad)} points, first {bad[:8]}"
    assert np.array_equal(got["kept_idx"], ref["kept_idx"]), what
    assert np.array_equal(got["ages"], fs.ages), what
    if _cv2() is not None:
        cvr = _circular(imgs, pts, ref_path.FeatureSet(), win, "cv2")["raw"]
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


def _eps_flip_cases(a, b, pts, want, win=21):
    """(start, epsilon) pairs whose track, at that epsilon, has an iteration where delta.ddot(delta) <= eps^2 (double, as
    OpenCV decides) and the float-only test (float)(dx^2 + dy^2) <= (float)eps^2 disagree.  At eps = 0.01 such an
    iteration is rarer than one in 10^8; choosing eps from a logged step makes one per start.  One case per start."""
    from oracle import cref
    _, _, _, log = cref.lk_track(a, b, pts, win=win, return_log=True)
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
        lg = cref.lk_track(a, b, p, win=win, epsilon=float(eps), return_log=True)[3]
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
def _level_sizes(w, h, nlev):
    sizes = []
    for l in range(nlev):
        sizes.append((w, h))
        w, h = (w + 1) // 2, (h + 1) // 2
    return sizes


def _outside(x, l, win, lw):
    """is the level-l origin floor(x * 2^-l - (W - 1) / 2), in float32 as the level-solve forms it, out of [-W, lw)?"""
    o = np.floor(np.float32(x) * np.float32(1.0 / (1 << l)) - np.float32((win - 1) * 0.5))
    return o < -win or o >= lw


def _bound_starts(w, h, nlev, win=21, shift=0.0):
    """At level l the I window's origin floor(x / 2^l - (W - 1) / 2) is in range (-W <= origin < lw) iff
    -(W + 1) / 2 * 2^l <= x < (lw + (W - 1) / 2) * 2^l: per level, axis (x with y mid-image, y with x mid-image) and
    bound v, the three starts v, the float just below v, and the first float below v (at most 64 ulps down) whose origin,
    rounded as the level-solve rounds it, lies on the other side of the edge from v's.  The float just below a lower
    bound can round back onto the edge once (W - 1) / 2 is subtracted; the third start then does cross it.  12 starts a
    level, in that order (_straddle_failures reads them so).  `shift` moves every bound by shift * 2^l (a wrong closed
    form, whose v and third start then do not straddle the edge)."""
    pts = []
    for l, (lw, lh) in enumerate(_level_sizes(w, h, nlev)):
        s = float(1 << l)
        lo = (-(win + 1) / 2 + shift) * s
        for hi, mid, axis, n in (((lw + (win - 1) / 2 + shift) * s, h / 2 + 0.3, 0, lw),
                                 ((lh + (win - 1) / 2 + shift) * s, w / 2 + 0.3, 1, lh)):
            for v in (lo, hi):
                v = np.float32(v)
                below = np.nextafter(v, np.float32(-np.inf))
                cross = below
                for _ in range(64):
                    if _outside(cross, l, win, n) != _outside(v, l, win, n):
                        break
                    cross = np.nextafter(cross, np.float32(-np.inf))
                else:
                    cross = below
                for x in (v, below, cross):
                    pts.append((x, mid) if axis == 0 else (mid, x))
    return np.array(pts, np.float32)


def _straddle_failures(a, b, pts, win, nlev):
    """The bounds of _bound_starts(..., nlev, win) whose first and third start do not straddle the edge in the oracle's
    log: at a lower bound v itself must reach the level-solve and the third start must get EV_IOUT at that level; at an
    upper bound the other way round.  Returns [(level, axis, "lo" / "hi")] of the bounds that fail."""
    from oracle import cref
    log = cref.lk_track(a, b, pts, win=win, return_log=True)[3]
    sel = log["kind"] == cref.EV_IOUT
    iout = set(zip(log["pt"][sel].tolist(), log["level"][sel].tolist()))
    bad = []
    for l in range(nlev):
        for axis in (0, 1):
            for k, side in enumerate(("lo", "hi")):
                p = 3 * ((l * 2 + axis) * 2 + k)
                at, cross = (p, l) in iout, (p + 2, l) in iout
                if (at, cross) != ((False, True) if side == "lo" else (True, False)):
                    bad.append((l, axis, side))
    return bad


def test_window_bound_starts(ctx):
    w, h = 1241, 376
    u = synth.stereo_unit(w, h, 31)
    imgs = [u[k] for k in ("l0", "r0", "l1", "r1")]
    pts = _bound_starts(w, h, 4)
    assert _straddle_failures(imgs[0], imgs[1], pts, 21, 4) == []
    # a start outside level 0 still carries the estimate of the coarser levels into its (status 0) output position
    _check_single(ctx, imgs[0], imgs[1], pts, "window bounds")
    _check_ring(ctx, imgs, pts, "window bounds ring")


# ---- pyramid depth -------------------------------------------------------------------------------------------------
# (w, h, levels): each side of the sizes where the coarsest level is 22 px (42/43, 84/85, 168/169), in width and in height
# separately; a one-level image; images narrower / shorter than the window
SIZES = [(42, 300, 1), (43, 300, 2), (84, 300, 2), (85, 300, 3), (168, 300, 3), (169, 300, 4),
         (500, 42, 1), (500, 43, 2), (500, 84, 2), (500, 85, 3), (500, 168, 3), (500, 169, 4),
         (40, 30, 1), (20, 200, 1), (200, 20, 1), (7, 60, 1), (60, 5, 1), (3, 3, 1)]
# k_lk_win: windows of each of its classes (all-tail 3, 4, 7; no tail 8, 16, 24, 32; SIMD + tail 9, 13, 17, 31)
WIN_WINDOWS = (3, 4, 7, 8, 9, 13, 16, 17, 24, 31, 32)


def _win_sizes(win):
    """(w, h, levels) at a window W: the pyramid stops once a level is not larger than W, so the depth changes between
    2^k W and 2^k W + 1 (k = 1..3), in width and in height separately (the other side never limits it); images narrower
    and shorter than the window, down to 3 x 3."""
    out = []
    for k in (1, 2, 3):
        out += [((1 << k) * win, 300, k), ((1 << k) * win + 1, 300, k + 1)]
        out += [(500, (1 << k) * win, k), (500, (1 << k) * win + 1, k + 1)]
    small = max(3, win - 1)
    out += [(small, 200, 1), (200, small, 1), (max(3, win // 2), max(3, win // 3), 1), (3, 3, 1)]
    return list(dict.fromkeys(out))


DEPTH_CASES = [pytest.param(21, w, h, n, id=f"{w}-{h}-{n}") for w, h, n in SIZES] + \
              [pytest.param(win, w, h, n, id=f"W{win}-{w}-{h}-{n}") for win in WIN_WINDOWS for w, h, n in _win_sizes(win)]


@pytest.fixture(scope="module")
def win_ctxs(built):
    """a context per window, made when first asked for"""
    from visual_odom_b200.capi import Context
    made = {}

    def get(win):
        if win not in made:
            made[win] = Context(0, max_features=8192, lk_win=win)
        return made[win]
    yield get
    for c in made.values():
        c.close()


@pytest.mark.parametrize("win,w,h,nlev", DEPTH_CASES)
def test_pyramid_depth_and_tiny_images(ctx, win_ctxs, win, w, h, nlev):
    from oracle import cref
    c = ctx if win == 21 else win_ctxs(win)
    u = synth.stereo_unit(1241, 376, 41)
    y0 = min(100, 376 - h)
    imgs = [np.ascontiguousarray(u[k][y0:y0 + h, 300:300 + w]) for k in ("l0", "r0", "l1", "r1")]
    assert imgs[0].shape == (h, w)
    assert cref.Pyramid(imgs[0], win).nlevels() == nlev
    rng = np.random.default_rng(w * 1000 + h)
    pts = np.concatenate([np.stack([rng.uniform(-25, w + 25, 300), rng.uniform(-25, h + 25, 300)], 1),
                          np.stack([rng.uniform(0, w, 200), rng.uniform(0, h, 200)], 1),
                          _bound_starts(w, h, nlev, win)]).astype(np.float32)
    _check_single(c, imgs[0], imgs[1], pts, f"W={win} {w}x{h}", win)
    _check_ring(c, imgs, pts, f"W={win} {w}x{h} ring", win)


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
