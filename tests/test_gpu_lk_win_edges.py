"""k_lk_win (csrc/lk_win.cu, every lk_win from 3 to 32 other than 21) at the edges of calcOpticalFlowPyrLK, bit for bit
against the oracle (oracle/lk_ref.c) and cv2, at windows of each of its three classes of float chain (nsimd = (W / 8) * 8):
all-tail (W < 8), no tail (W % 8 == 0, W = 32 reading the outermost padded column and row) and SIMD + tail (the others).

- the mined window-edge fixture (tests/golden/lk_win_edges/lk_win_edges.npz, made by tests/golden/make_lk_edges.py
  --windows) through vo_lk_track and vo_circular_match on a fresh context per window, with the SM partition at 0 and 8 (the
  single-call entry points run no CUDA graph, so the graphs option does not reach them).  k_lk_win has no exact-integer
  path: every bit of b is the order of its float chains, and tests/test_oracle_lk_win_edges.py shows that each wrong
  order of them that applies at a window changes a stored output;
- window-bound starts in closed form, each bound's pair straddling its edge in the oracle's event log;
- the convergence test decided in double, host images whose row pitch is not their width, and err not requested;
- consecutive calls on one context at the work queue's boundaries (1, 4 and 5 items, and one below, at and above the
  resident warp count), which hold only if the last retiring warp resets the queue for the next launch.

tests/test_gpu_lk_edges.py runs the pyramid-depth transitions and images smaller than the window at these windows.
The SIZED instantiation k_lk_win<true> is not reached here: no entry point gives it caller-chosen starts, so the sized
multi-sequence tests (test_gpu_lk_windows.py::test_mseq_two_sizes_each_as_run_alone) stay its only check."""
import json
import os
import sys

import numpy as np
import pytest

from visual_odom_b200 import synth

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_lk_edges as mk          # noqa: E402
import test_gpu_lk_edges as E       # noqa: E402

WINDOWS = E.WIN_WINDOWS
PARTITIONS = (0, 8)


def _wid(win):
    return f"W{win}-{mk.window_class(win)}"


def _context(win, opts=None, **params):
    from visual_odom_b200.capi import Context
    c = Context(0, lk_win=win, **dict(dict(max_features=8192), **params))
    try:
        for k, v in (opts or {}).items():
            c.set_option(k, v)
    except Exception:
        c.close()
        raise
    return c


def _tags_of(tags, idx):
    return [[t for t in mk.TAGS if tags[i] & mk.BIT[t]] for i in idx[:8]]


# ---- the mined fixture ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def win_edges(built):
    fx = np.load(mk.WIN_OUT)
    assert tuple(json.loads(str(fx["windows"]))) == mk.WIN_WINDOWS
    imgs = []
    for ri, r in enumerate(json.loads(str(fx["recipes"]))):
        im = mk.images(r)
        assert [mk.sha(a) for a in im] == json.loads(str(fx[f"sha256_{ri}"]))
        imgs.append(im)
    return fx, imgs


@pytest.mark.parametrize("part", PARTITIONS, ids=[f"partition{p}" for p in PARTITIONS])
@pytest.mark.parametrize("win", mk.WIN_WINDOWS, ids=[_wid(w) for w in mk.WIN_WINDOWS])
def test_win_edge_fixture_bit_exact(win_edges, win, part):
    """The fixture's starts at one window (stored outputs = cv2 = oracle): call L0 -> R0 through vo_lk_track, the ring
    through vo_circular_match.  A mismatch names the starts and the categories they were mined for."""
    fx, imgs = win_edges
    c = _context(win, dict(sm_partition=part))
    try:
        for ri, im in enumerate(imgs):
            g = lambda name: fx[mk.win_key(f"{name}_{ri}", win)]
            pts, tags, out, status, err = g("pts"), g("tags"), g("out"), g("status"), g("err")
            go, gs, ge = c.lk_track(im[0], im[1], pts)
            bad = np.nonzero((go != out[0]).any(1) | (gs != status[0]))[0]
            assert len(bad) == 0, f"W={win} recipe {ri} single call differs at {bad[:8]}, tags {_tags_of(tags, bad)}"
            E._assert_single((go, gs, ge), (out[0], status[0], err[0]), f"W={win} recipe {ri} single call")
            got = c.circular_match(*im, pts)
            for k in range(4):
                bad = np.nonzero((got["raw4"][k] != out[k]).any(1) | (got["status4"][k] != status[k]))[0]
                assert len(bad) == 0, f"W={win} recipe {ri}: ring call {k} differs at {bad[:8]}, tags {_tags_of(tags, bad)}"
    finally:
        c.close()


# ---- window-bound starts in closed form ----------------------------------------------------------------------------
def _outermost_reads(pts, log, win, sizes):
    """Which outermost padded lines of a level the starts' I windows read with a nonzero bilinear weight, from the
    origins in the oracle's log (level-solve set-ups): "left" (ipx = -W, column -W), "right" (ipx = lw - 1 with a nonzero
    right tap, column lw - 1 + W), "top", "bottom" likewise for rows."""
    from oracle import cref
    st = log[(log["kind"] == cref.EV_SETUP) | (log["kind"] == cref.EV_REJECT)]
    seen = set()
    for ev in st:
        l = int(ev["level"])
        lw, lh = sizes[l]
        p = pts[ev["pt"]] * np.float32(1.0 / (1 << l)) - np.float32((win - 1) * 0.5)
        a, b = p[0] - np.float32(ev["ipx"]), p[1] - np.float32(ev["ipy"])
        one, scale = np.float32(1), np.float32(1 << 14)
        w01 = np.rint(a * (one - b) * scale)
        w10 = np.rint((one - a) * b * scale)
        w00 = np.rint((one - a) * (one - b) * scale)
        w11 = 16384 - w00 - w01 - w10
        if ev["ipx"] == -win and w00 + w10 > 0:
            seen.add("left")
        if ev["ipx"] == lw - 1 and w01 + w11 > 0:
            seen.add("right")
        if ev["ipy"] == -win and w00 + w01 > 0:
            seen.add("top")
        if ev["ipy"] == lh - 1 and w10 + w11 > 0:
            seen.add("bottom")
    return seen


@pytest.mark.parametrize("win", WINDOWS, ids=[_wid(w) for w in WINDOWS])
def test_window_bound_starts(built, win):
    """Every bound's starts straddle its edge in the oracle's log; at W = 32 some start reads the outermost padded column
    and row on each side (VO_PAD = 32); the single call and the ring equal the oracle and cv2."""
    from oracle import cref
    w, h = 1241, 376
    u = synth.stereo_unit(w, h, 31)
    imgs = [u[k] for k in ("l0", "r0", "l1", "r1")]
    nlev = cref.Pyramid(imgs[0], win).nlevels()
    pts = E._bound_starts(w, h, nlev, win)
    assert E._straddle_failures(imgs[0], imgs[1], pts, win, nlev) == []
    if win == 32:
        log = cref.lk_track(imgs[0], imgs[1], pts, win=win, return_log=True)[3]
        assert _outermost_reads(pts, log, win, E._level_sizes(w, h, nlev)) == {"left", "right", "top", "bottom"}
    c = _context(win)
    try:
        E._check_single(c, imgs[0], imgs[1], pts, f"window bounds W={win}", win)
        E._check_ring(c, imgs, pts, f"window bounds ring W={win}", win)
    finally:
        c.close()


# ---- the convergence test decided in double ------------------------------------------------------------------------
@pytest.mark.parametrize("win", WINDOWS, ids=[_wid(w) for w in WINDOWS])
def test_eps_decided_in_double(built, win):
    """Contexts whose lk_epsilon puts an iteration between the double and the float form of the convergence test."""
    from oracle import cref
    u = synth.stereo_unit(1241, 376, 5)
    corners, _ = cref.fast_detect(u["l0"])
    cases = E._eps_flip_cases(u["l0"], u["r0"], synth.select_features(corners, 600), 4, win)
    assert len(cases) == 4
    for p, eps in cases:
        c = _context(win, max_features=64, lk_epsilon=eps)
        try:
            got = c.lk_track(u["l0"], u["r0"], p)
        finally:
            c.close()
        what = f"W={win} eps {eps!r} at {p[0]}"
        E._assert_single(got, cref.lk_track(u["l0"], u["r0"], p, win=win, epsilon=eps), what)
        cv2 = E._cv2()
        if cv2 is not None:
            crit = (cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, 30, eps)
            o, s, e = cv2.calcOpticalFlowPyrLK(u["l0"], u["r0"], p.reshape(-1, 1, 2), None, winSize=(win, win),
                                               maxLevel=3, criteria=crit, flags=0, minEigThreshold=0.001)
            E._assert_single(got, (o.reshape(-1, 2), s.ravel(), e.ravel()), f"{what} vs cv2")


# ---- host images whose pitch is not their width, err not requested --------------------------------------------------
@pytest.mark.parametrize("win", WINDOWS, ids=[_wid(w) for w in WINDOWS])
def test_row_pitch_not_width(built, win):
    from oracle import cref
    w, h = 333, 129
    u = synth.stereo_unit(w, h, 13, scene="v0")
    imgs = []
    for k in ("l0", "r0", "l1", "r1"):
        wide = np.zeros((h, w + 45), np.uint8)
        wide[:, 7:7 + w] = u[k]
        imgs.append(wide[:, 7:7 + w])          # a view: row pitch w + 45, passed as the C-ABI pitch
    assert imgs[0].strides == (w + 45, 1) and not imgs[0].flags.c_contiguous
    corners, _ = cref.fast_detect(u["l0"])
    nlev = cref.Pyramid(u["l0"], win).nlevels()
    pts = np.concatenate([synth.select_features(corners, 400), E._bound_starts(w, h, nlev, win)]).astype(np.float32)
    ref, cvr = E._single_refs(u["l0"], u["r0"], pts, win)
    c = _context(win)
    try:
        got = c.lk_track(imgs[0], imgs[1], pts)
        E._assert_single(got, ref, f"W={win} pitched single call")
        if cvr is not None:
            E._assert_single(got, cvr, f"W={win} pitched single call vs cv2")
        E._check_ring(c, imgs, pts, f"W={win} pitched ring", win)
    finally:
        c.close()


@pytest.mark.parametrize("win", WINDOWS, ids=[_wid(w) for w in WINDOWS])
def test_status_without_err(built, win):
    """err not requested: positions and status are those of the call that requests it (which equals the oracle)."""
    from oracle import cref
    u = synth.stereo_unit(1241, 376, 31)
    nlev = cref.Pyramid(u["l0"], win).nlevels()
    corners, _ = cref.fast_detect(u["l0"])
    pts = np.concatenate([synth.select_features(corners, 500), E._bound_starts(1241, 376, nlev, win)]).astype(np.float32)
    c = _context(win)
    try:
        E._check_single(c, u["l0"], u["r0"], pts, f"W={win} with err", win)
        go, gs, _ = c.lk_track(u["l0"], u["r0"], pts)
        no, ns, ne = c.lk_track(u["l0"], u["r0"], pts, want_err=False)
    finally:
        c.close()
    assert ne is None and np.array_equal(ns, gs) and np.array_equal(no, go)


# ---- consecutive calls at the work queue's boundaries --------------------------------------------------------------
LKW_WARPS = 6 * 4                   # lk_win.cu: LKW_CTAS_PER_SM x LKW_WARPS_PER_CTA resident warps per SM


@pytest.mark.parametrize("part", PARTITIONS, ids=[f"partition{p}" for p in PARTITIONS])
@pytest.mark.parametrize("win", (4, 13, 32), ids=[_wid(w) for w in (4, 13, 32)])
def test_consecutive_calls_at_queue_boundaries(built, win, part):
    """vo_launch_lk_win launches ceil(items / 4) CTAs of 4 warps, at most the resident ones; each warp takes work items
    from a queue that the last warp to retire resets.  Calls of 1, 4, 5, R - 1, R and R + 1 items (R the resident warp
    count), alternating vo_lk_track and vo_circular_match on two sets of starts, each equal to the oracle: a queue left
    unreset skips the next launch's items and leaves the previous call's outputs."""
    torch = pytest.importorskip("torch")
    from oracle import cref, ref_path
    import lk_window_scenes as S
    resident = torch.cuda.get_device_properties(0).multi_processor_count * LKW_WARPS
    counts = (1, 4, 5, resident - 1, resident, resident + 1, 5, 1)
    u = synth.stereo_unit(1241, 376, 17)
    imgs = [u[k] for k in ("l0", "r0", "l1", "r1")]
    rng = np.random.default_rng(win)
    n = resident + 1
    pools = [np.stack([rng.uniform(-20, 1261, n), rng.uniform(-20, 396, n)], 1).astype(np.float32) for _ in range(2)]
    # LK tracks every start on its own, so the oracle's outputs on a prefix of the starts are a prefix of its outputs
    single = cref.lk_track(imgs[0], imgs[1], pools[0], win=win)
    ring = S.circular_matching(*imgs, pools[1], ref_path.FeatureSet(), win, "c")["raw"]
    c = _context(win, dict(sm_partition=part), max_features=n + 64)
    try:
        for k in counts:
            got = c.lk_track(imgs[0], imgs[1], pools[0][:k])
            E._assert_single(got, tuple(r[:k] for r in single), f"W={win} partition {part}: vo_lk_track of {k} starts")
            got = c.circular_match(*imgs, pools[1][:k])
            assert np.array_equal(got["status4"], ring["status"][:, :k]), f"W={win}: ring of {k} starts, status"
            for q, name in enumerate(("r0", "r1", "l1", "l0_ret")):
                bad = np.nonzero((got["raw4"][q] != ring[name][:k]).any(1))[0]
                assert len(bad) == 0, f"W={win} partition {part}: ring of {k} starts, call {q} differs at {bad[:8]}"
    finally:
        c.close()
