"""The LK window-edge fixture (tests/golden/lk_win_edges/lk_win_edges.npz, made by tests/golden/make_lk_edges.py --windows)
on the CPU, at each mined window: the images are regenerated bit for bit; cv2 and the oracle agree with the stored outputs
of the single call and of the four ring calls; every category holds its starts, re-derived from the oracle's log; and
every wrong summation rule that applies at a window changes a stored output there, while the others change nothing.
Also the closed form of the window-bound starts (tests/test_gpu_lk_edges.py) at every window of k_lk_win's classes: each
bound's starts straddle the edge in the oracle's log, and a closed form off by half a pixel does not."""
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_lk_edges as mk          # noqa: E402
import test_gpu_lk_edges as E       # noqa: E402

cref = mk.cref
IDS = [f"W{w}-{mk.window_class(w)}" for w in mk.WIN_WINDOWS]
# per recipe: category -> the least number of starts within mk.WITHIN, at every mined window
QUOTA = [dict(HALF=5, EPS=3, CAP=5, JOUT0=3, JOUTC=3, FINAL=3), dict(MINEIG=2)]


@pytest.fixture(scope="module")
def fx(built):
    return np.load(mk.WIN_OUT)


@pytest.fixture(scope="module")
def images(fx):
    return [mk.images(r) for r in json.loads(str(fx["recipes"]))]


@pytest.fixture(scope="module")
def runs(fx, images):
    """per window and recipe: starts, stored arrays and the oracle's ring (out, status, err, log per call)"""
    out = {}
    for win in mk.WIN_WINDOWS:
        for ri, imgs in enumerate(images):
            g = {k: fx[mk.win_key(f"{k}_{ri}", win)] for k in ("pts", "tags", "out", "status", "err")}
            out[win, ri] = dict(g, imgs=imgs, ring=mk.ring_oracle(imgs, g["pts"], win=win))
    return out


def test_images_match_recorded_hashes(fx, images):
    assert tuple(json.loads(str(fx["windows"]))) == mk.WIN_WINDOWS
    for ri, imgs in enumerate(images):
        assert [mk.sha(a) for a in imgs] == json.loads(str(fx[f"sha256_{ri}"]))


@pytest.mark.parametrize("win", mk.WIN_WINDOWS, ids=IDS)
def test_oracle_matches_stored_outputs(runs, win):
    """The four ring calls, and the single call L0 -> R0 on its own."""
    for ri in (0, 1):
        run = runs[win, ri]
        s, o, e = run["status"], run["out"], run["err"]
        for k, (ok, sk, ek, _) in enumerate(run["ring"]):
            assert np.array_equal(sk, s[k]), (win, ri, k)
            assert np.array_equal(ok, o[k]), (win, ri, k)
            assert np.array_equal(ek[sk == 1], e[k][sk == 1]), (win, ri, k)
        o1, s1, e1 = cref.lk_track(run["imgs"][0], run["imgs"][1], run["pts"], win=win)
        assert np.array_equal(s1, s[0]) and np.array_equal(o1, o[0]), (win, ri)
        assert np.array_equal(e1[s1 == 1], e[0][s1 == 1]), (win, ri)


@pytest.mark.parametrize("win", mk.WIN_WINDOWS, ids=IDS)
def test_cv2_matches_stored_outputs(runs, win):
    cv2 = pytest.importorskip("cv2")
    crit = (cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, 30, 0.01)
    for ri in (0, 1):
        run = runs[win, ri]
        o, s, e = mk.ring_cv2(run["imgs"], run["pts"], win)
        assert np.array_equal(s, run["status"]) and np.array_equal(o, run["out"]), (win, ri)
        assert np.array_equal(np.where(s == 1, e, 0), run["err"]), (win, ri)
        o1, s1, _ = cv2.calcOpticalFlowPyrLK(run["imgs"][0], run["imgs"][1], run["pts"].reshape(-1, 1, 2), None,
                                             winSize=(win, win), maxLevel=3, criteria=crit, flags=0,
                                             minEigThreshold=0.001)
        assert np.array_equal(o1.reshape(-1, 2), o[0]) and np.array_equal(s1.ravel(), s[0]), (win, ri)


@pytest.mark.parametrize("win", mk.WIN_WINDOWS, ids=IDS)
def test_categories_hold_their_points(fx, runs, win):
    assert tuple(json.loads(str(fx["tags"]))) == mk.TAGS
    for ri in (0, 1):
        run = runs[win, ri]
        m = mk.point_margins([r[3] for r in run["ring"]], len(run["pts"]))
        for t in mk.TAGS:
            hit = m[t] <= mk.WITHIN[t]
            assert np.array_equal(hit, (run["tags"] & mk.BIT[t]) != 0), (win, ri, t)
            print(f"W={win} recipe {ri} {t:6s}: {int(hit.sum()):3d} starts within {mk.WITHIN[t]}, closest {m[t].min():.3g}")
        for t, q in QUOTA[ri].items():
            assert (m[t] <= mk.WITHIN[t]).sum() >= q, (win, ri, t)


def test_min_eig_threshold_sampled_on_both_sides(runs):
    """At every mined window some contrast-reduced start's level-0 minEig lies within 8 ulps of 0.001f below it (rejected)
    and some at or above it (kept)."""
    for win in mk.WIN_WINDOWS:
        log = runs[win, 1]["ring"][0][3]
        st = log[((log["kind"] == cref.EV_SETUP) | (log["kind"] == cref.EV_REJECT)) & (log["level"] == 0)]
        u = mk.ulps(st["min_eig"], mk.THR)
        near = np.abs(u) <= 8
        rejected = st["kind"] == cref.EV_REJECT
        assert np.array_equal(rejected[near], u[near] < 0), win
        assert (near & rejected).any() and (near & ~rejected).any(), win


# ---- the wrong summation rules ---------------------------------------------------------------------------------------
def test_applicability_matrix():
    """The matrix written into the mining script is applies() at the mined windows, and those windows cover the three
    classes of k_lk_win's float chains."""
    assert {w: tuple(r for r in mk.RULES if mk.applies(r, w)) for w in mk.WIN_WINDOWS} == mk.APPLIES
    assert {mk.window_class(w) for w in mk.WIN_WINDOWS} == {"all-tail", "no-tail", "simd+tail"}
    # the classes at the windows they are named for
    assert [mk.window_class(w) for w in (3, 7, 8, 24, 9, 31)] == ["all-tail"] * 2 + ["no-tail"] * 2 + ["simd+tail"] * 2


PAIRS = [(w, r) for w in mk.WIN_WINDOWS for r in mk.APPLIES[w]]


@pytest.mark.parametrize("win,rule", PAIRS, ids=[f"W{w}-{mk.window_class(w)}-{r}" for w, r in PAIRS])
def test_wrong_rule_changes_a_stored_output(runs, win, rule):
    """Each wrong rule that applies at a window changes a position or a status of the fixture's ring there."""
    run = runs[win, 0]
    changed = mk.ring_changed(run["imgs"], run["pts"], mk.RULES[rule], run["ring"], win)
    print(f"W={win} {rule}: {int(changed.sum())} of {len(changed)} starts changed")
    assert changed.any(), (win, rule)


@pytest.mark.parametrize("win", mk.WIN_WINDOWS, ids=IDS)
def test_kernel_rule_and_inapplicable_rules_change_nothing(runs, win):
    """The oracle forming b as k_lk_win does (SUM_WIN) is cv2; so is every wrong rule that does not apply at the window."""
    for ri in (0, 1):
        run = runs[win, ri]
        for rule in ["WIN"] + [r for r in mk.RULES if r not in mk.APPLIES[win]]:
            mode = cref.SUM_WIN if rule == "WIN" else mk.RULES[rule]
            assert not mk.ring_changed(run["imgs"], run["pts"], mode, run["ring"], win).any(), (win, ri, rule)


# ---- window-bound starts in closed form ----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bound_scene(built):
    from visual_odom_b200 import synth
    u = synth.stereo_unit(1241, 376, 31)
    return u["l0"], u["r0"]


@pytest.mark.parametrize("win", E.WIN_WINDOWS + (21,))
def test_bound_starts_straddle_their_edges(bound_scene, win):
    """Per level, axis and bound, one start reaches the level-solve and the other gets EV_IOUT at that level; moving
    the closed form by half a pixel either way breaks that at every bound."""
    a, b = bound_scene
    nlev = cref.Pyramid(a, win).nlevels()
    assert E._straddle_failures(a, b, E._bound_starts(1241, 376, nlev, win), win, nlev) == []
    for shift in (0.5, -0.5):
        assert len(E._straddle_failures(a, b, E._bound_starts(1241, 376, nlev, win, shift), win, nlev)) == 4 * nlev


def test_bound_starts_at_21_hold_the_previous_starts(built):
    """At W = 21 the closed form gives the starts the 21 x 21 tests used before it took a window (the bound and the float
    below it, -11 * 2^l and (lw + 10) * 2^l), and beside them the first float that crosses the edge as the level-solve
    rounds it."""
    w, h, nlev = 1241, 376, 4
    pts = E._bound_starts(w, h, nlev).reshape(-1, 3, 2)
    old = []
    for l, (lw, lh) in enumerate(E._level_sizes(w, h, nlev)):
        s = float(1 << l)
        for lo, hi, mid, axis in ((-11 * s, (lw + 10) * s, h / 2 + 0.3, 0), (-11 * s, (lh + 10) * s, w / 2 + 0.3, 1)):
            for v in (lo, hi):
                for x in (np.float32(v), np.nextafter(np.float32(v), np.float32(-np.inf))):
                    old.append((x, mid) if axis == 0 else (mid, x))
    assert np.array_equal(pts[:, :2].reshape(-1, 2), np.array(old, np.float32))
