"""The LK edge fixture (tests/golden/lk_edges/lk_edges.npz, made by tests/golden/make_lk_edges.py) on the CPU: the images it was
mined on are regenerated bit for bit, cv2 and the oracle still agree with the stored outputs on every point, every
category still holds its points within its margin, and the margins are tight enough that a one-rounding change of a
decision would change an output."""
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_lk_edges as mk          # noqa: E402

FIXTURE = os.path.join(HERE, "golden", "lk_edges", "lk_edges.npz")
# per recipe: category -> the least number of points within mk.WITHIN
QUOTA = [dict(HALF=5, EPS=5, CAP=5, JOUT0=3, JOUTC=3, FINAL=3), dict(MINEIG=10)]


@pytest.fixture(scope="module")
def fx(built):
    return np.load(FIXTURE)


@pytest.fixture(scope="module")
def runs(fx):
    """per recipe: images, points and the oracle's ring (out, status, err, log per call)"""
    out = []
    for ri, r in enumerate(json.loads(str(fx["recipes"]))):
        imgs = mk.images(r)
        pts = fx[f"pts_{ri}"]
        out.append(dict(imgs=imgs, pts=pts, ring=mk.ring_oracle(imgs, pts)))
    return out


def test_images_match_recorded_hashes(fx):
    for ri, r in enumerate(json.loads(str(fx["recipes"]))):
        assert [mk.sha(a) for a in mk.images(r)] == json.loads(str(fx[f"sha256_{ri}"]))


def test_oracle_matches_stored_outputs(fx, runs):
    for ri, run in enumerate(runs):
        s = fx[f"status_{ri}"]
        for k, (o, st, e, _) in enumerate(run["ring"]):
            assert np.array_equal(st, s[k]), (ri, k)
            assert np.array_equal(o, fx[f"out_{ri}"][k]), (ri, k)
            assert np.array_equal(e[st == 1], fx[f"err_{ri}"][k][st == 1]), (ri, k)


def test_cv2_matches_stored_outputs(fx, runs):
    pytest.importorskip("cv2")
    for ri, run in enumerate(runs):
        o, s, e = mk.ring_cv2(run["imgs"], run["pts"])
        assert np.array_equal(s, fx[f"status_{ri}"])
        assert np.array_equal(o, fx[f"out_{ri}"])
        assert np.array_equal(np.where(s == 1, e, 0), fx[f"err_{ri}"])


def test_categories_hold_their_points(fx, runs):
    tags = json.loads(str(fx["tags"]))
    assert tuple(tags) == mk.TAGS
    for ri, run in enumerate(runs):
        m = mk.point_margins([r[3] for r in run["ring"]], len(run["pts"]))
        stored = fx[f"tags_{ri}"]
        for t in mk.TAGS:
            hit = m[t] <= mk.WITHIN[t]
            assert np.array_equal(hit, (stored & mk.BIT[t]) != 0), (ri, t)
            print(f"recipe {ri} {t:6s}: {int(hit.sum()):3d} points within {mk.WITHIN[t]}, closest {m[t].min():.3g}")
        for t, q in QUOTA[ri].items():
            assert (m[t] <= mk.WITHIN[t]).sum() >= q, (ri, t)


def _level0_setups(run):
    log = run["ring"][0][3]
    return log[((log["kind"] == mk.cref.EV_SETUP) | (log["kind"] == mk.cref.EV_REJECT)) & (log["level"] == 0)]


def test_min_eig_threshold_is_sampled_at_the_float_edge(runs):
    """Level-0 minEig of the contrast-reduced starts: both outcomes within 8 ulps of 0.001f, 0.001f itself (accepted) and
    the float just below it (rejected).  Changing minEig by one ulp, or comparing minEig <= 0.001f, changes a status."""
    st = _level0_setups(runs[1])
    u = mk.ulps(st["min_eig"], mk.THR)
    near = np.abs(u) <= 8
    rejected = st["kind"] == mk.cref.EV_REJECT
    assert np.array_equal(rejected[near], u[near] < 0)
    assert (near & ~rejected).sum() >= 5 and (near & rejected).sum() >= 5
    assert (u == 0).any() and (u == -1).any()
    me = st["min_eig"]
    thr = 1e-3
    for changed in (np.nextafter(me, np.float32(1)), np.nextafter(me, np.float32(0))):
        assert ((changed.astype(np.float64) < thr) != rejected).any()
    assert ((me <= mk.THR) != rejected).any()
    # a rejection at level 0 is a cleared status of the first call
    s0 = runs[1]["ring"][0][1]
    assert (s0[st["pt"][near & rejected]] == 0).all()


def test_half_step_and_eps_margins(runs):
    """The half-step sums reach 0.01f within a few ulps on both sides; ||delta||^2 reaches the +-1e-6 band around eps^2
    in which the GPU kernel decides in double.  Reported: how many of those iterations a float-only test would flip."""
    log = np.concatenate([r[3] for r in runs[0]["ring"]])
    it = log[np.isin(log["kind"], mk.ITER_KINDS) & (log["iter"] > 0)]
    for comp in ("sdx", "sdy"):
        u = mk.ulps(it[comp], mk.HALF_F)
        print(f"{comp}: closest ulps to 0.01f below {u[u <= 0].max() if (u <= 0).any() else None}, "
              f"above {u[u > 0].min() if (u > 0).any() else None}")
    u = np.concatenate([mk.ulps(it["sdx"], mk.HALF_F), mk.ulps(it["sdy"], mk.HALF_F)])
    assert ((u <= 0) & (u >= -64)).any() and ((u > 0) & (u <= 64)).any()
    all_it = log[np.isin(log["kind"], mk.ITER_KINDS)]
    band = np.abs(all_it["d2f"].astype(np.float64) / mk.EPS2 - 1) <= 1e-6
    flip = (all_it["d2f"] <= np.float32(mk.EPS2)) != (all_it["d2"] <= mk.EPS2)
    print(f"eps^2: {int(band.sum())} iterations in the +-1e-6 band, {int(flip.sum())} decided differently in float")
    assert band.sum() >= 5
    assert (all_it["d2"][band] <= mk.EPS2).any() and (all_it["d2"][band] > mk.EPS2).any()
