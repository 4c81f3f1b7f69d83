"""The LK sum-edge fixture (tests/golden/lk_sum_edges/lk_sum_edges.npz, made by tests/golden/make_lk_sum_edges.py) on the
CPU: the images it was mined on are regenerated bit for bit; cv2 and the oracle agree with the stored outputs on every
start; every category holds its starts, re-derived from the oracle's log; k_lk_ring's vote is sound on the fixture and
on the benchmark scene; and each wrong vote or combination order changes an output of the fixture."""
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_lk_sum_edges as ms      # noqa: E402

mk = ms.mk
cref = ms.cref
# per recipe: category -> the least number of starts within ms.WITHIN
QUOTA = dict(VOTE_IN=8, VOTE_OUT=8, TAIL_ONLY=6, B2_ONLY=6, COMBINE=8)


@pytest.fixture(scope="module")
def fx(built):
    return np.load(ms.OUT)


@pytest.fixture(scope="module")
def runs(fx):
    """per recipe: images, starts, stored tags and the oracle's ring (out, status, err, log per call)"""
    out = []
    for ri, r in enumerate(json.loads(str(fx["recipes"]))):
        imgs = mk.images(r)
        pts = fx[f"pts_{ri}"]
        out.append(dict(imgs=imgs, pts=pts, tags=fx[f"tags_{ri}"], ring=mk.ring_oracle(imgs, pts)))
    return out


@pytest.fixture(scope="module")
def bench_scene(built):
    """The benchmark scene, stereo_unit(1241, 376, 0) with 2000 FAST features, and the oracle's ring on it."""
    from visual_odom_b200 import synth
    u = synth.stereo_unit(1241, 376, 0, cal=synth.KITTI00)
    imgs = [u[k] for k in ("l0", "r0", "l1", "r1")]
    corners, _ = cref.fast_detect(imgs[0])
    pts = synth.select_features(corners, 2000)
    return dict(imgs=imgs, pts=pts, ring=mk.ring_oracle(imgs, pts))


def test_images_match_recorded_hashes(fx):
    for ri, r in enumerate(json.loads(str(fx["recipes"]))):
        assert [mk.sha(a) for a in mk.images(r)] == json.loads(str(fx[f"sha256_{ri}"]))


def test_oracle_matches_stored_outputs(fx, runs):
    """The four ring calls, and the single call L0 -> R0 on its own."""
    for ri, run in enumerate(runs):
        s, o, e = fx[f"status_{ri}"], fx[f"out_{ri}"], fx[f"err_{ri}"]
        for k, (ok, sk, ek, _) in enumerate(run["ring"]):
            assert np.array_equal(sk, s[k]), (ri, k)
            assert np.array_equal(ok, o[k]), (ri, k)
            assert np.array_equal(ek[sk == 1], e[k][sk == 1]), (ri, k)
        o1, s1, e1 = cref.lk_track(run["imgs"][0], run["imgs"][1], run["pts"])
        assert np.array_equal(s1, s[0]) and np.array_equal(o1, o[0]), ri
        assert np.array_equal(e1[s1 == 1], e[0][s1 == 1]), ri


def test_cv2_matches_stored_outputs(fx, runs):
    cv2 = pytest.importorskip("cv2")
    crit = (cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, 30, 0.01)
    for ri, run in enumerate(runs):
        o, s, e = mk.ring_cv2(run["imgs"], run["pts"])
        assert np.array_equal(s, fx[f"status_{ri}"])
        assert np.array_equal(o, fx[f"out_{ri}"])
        assert np.array_equal(np.where(s == 1, e, 0), fx[f"err_{ri}"])
        o1, s1, e1 = cv2.calcOpticalFlowPyrLK(run["imgs"][0], run["imgs"][1], run["pts"].reshape(-1, 1, 2), None,
                                              winSize=(21, 21), maxLevel=3, criteria=crit, flags=0,
                                              minEigThreshold=0.001)
        assert np.array_equal(o1.reshape(-1, 2), o[0]) and np.array_equal(s1.ravel(), s[0]), ri


def test_categories_hold_their_points(fx, runs):
    assert tuple(json.loads(str(fx["tags"]))) == ms.TAGS
    for ri, run in enumerate(runs):
        m, side = ms.point_margins([r[3] for r in run["ring"]], len(run["pts"]))
        for t in ms.TAGS:
            hit = m[t] <= ms.WITHIN[t]
            assert np.array_equal(hit, (run["tags"] & ms.BIT[t]) != 0), (ri, t)
            print(f"recipe {ri} {t:9s}: {int(hit.sum()):3d} starts, closest {m[t].min() * ms.LIM:.0f}")
            assert hit.sum() >= QUOTA[t], (ri, t)
        # VOTE_IN on both quantities, and close to the bound from below (within 2^24 / 10^4)
        vin = m["VOTE_IN"] <= ms.WITHIN["VOTE_IN"]
        assert (vin & (side == 0)).sum() >= QUOTA["VOTE_IN"] // 2 and (vin & (side == 1)).sum() >= QUOTA["VOTE_IN"] // 2
        assert 0 <= m["VOTE_IN"].min() * ms.LIM <= 100, ri


def test_vote_margins_from_the_log(runs):
    """The margins re-derived from P and N: VOTE_IN iterations do pass max(P, N) <= 2^24 with every prefix exact;
    VOTE_OUT iterations sit above it, within twice the bound, with a float chain off its integer total; TAIL_ONLY and
    B2_ONLY iterations fail on a tail chain / a b2 chain only."""
    for ri, run in enumerate(runs):
        for log in (r[3] for r in run["ring"]):
            t = ms.iterations(log)
            it, pn, vot = t["it"], t["pn"], t["voted"]
            top = pn.max(1)
            inn = vot & (top <= ms.LIM) & (top >= ms.LIM * (1 - ms.WITHIN["VOTE_IN"]))
            assert (it["maxpre"][inn] <= ms.LIM).all() and (it["maxadd"][inn] <= ms.LIM).all()
            assert (it["fchain"][inn] == it["total"][inn]).all()
            out = vot & (top > ms.LIM) & (top <= ms.LIM * (1 + ms.WITHIN["VOTE_OUT"])) & ~t["fsame"].all(1)
            # a chain whose float differs is a chain that left the bound, and one of its prefixes did
            bad = ~t["fsame"][out]
            assert (pn[out][bad] > ms.LIM).all() and (it["maxpre"][out][bad] > ms.LIM).all()
            assert ((it["pos"] - it["neg"]) == it["total"]).all() and ((it["pos"] + it["neg"]) == it["sabs"]).all()


def _unsound(ring):
    """(iterations, iterations the kernel's vote accepts, accepted ones with a prefix or an addend beyond +-2^24)"""
    n = acc = bad = 0
    for r in ring:
        t = ms.iterations(r[3])
        it, a = t["it"], t["accept"]
        n += len(it); acc += int(a.sum())
        bad += int((a & ((it["maxpre"] > ms.LIM).any(1) | (it["maxadd"] > ms.LIM).any(1))).sum())
    return n, acc, bad


def test_vote_is_sound(runs, bench_scene):
    """No iteration that k_lk_ring's vote accepts has a chain prefix or addend beyond +-2^24, on the fixture and on the
    benchmark scene; and the oracle taking the kernel's two paths (SUM_KERNEL) equals cv2 there."""
    for what, run in [(f"recipe {ri}", r) for ri, r in enumerate(runs)] + [("benchmark scene", bench_scene)]:
        n, acc, bad = _unsound(run["ring"])
        print(f"{what}: {n} Newton iterations, the vote accepts {100.0 * acc / n:.1f} %, unsound {bad}")
        assert bad == 0 and acc > 0, what
        changed = ms.ring_changed(run["imgs"], run["pts"], cref.SUM_KERNEL, run["ring"])
        assert not changed.any(), f"{what}: the kernel's sum paths differ from cv2 at {np.nonzero(changed)[0][:8]}"


@pytest.mark.parametrize("mode", sorted(ms.CATCHES), ids=[f"M{m - cref.SUM_KERNEL}" for m in sorted(ms.CATCHES)])
def test_wrong_sum_rule_changes_a_fixture_output(runs, mode):
    """Each wrong rule changes the ring of at least one start of each recipe, among the starts of the category that
    catches it (ms.CATCHES: M1 / M2 by VOTE_OUT, M3 / M6 by TAIL_ONLY, M4 by B2_ONLY, M5 by COMBINE)."""
    cat = ms.CATCHES[mode]
    for ri, run in enumerate(runs):
        changed = ms.ring_changed(run["imgs"], run["pts"], mode, run["ring"])
        caught = changed & ((run["tags"] & ms.BIT[cat]) != 0)
        print(f"M{mode - cref.SUM_KERNEL} recipe {ri}: {int(changed.sum())} starts changed, {int(caught.sum())} of {cat}")
        assert caught.any(), (ri, cat)
