"""Mines tests/golden/lk_edges/lk_edges.npz (the 21 x 21 window of k_lk_ring) and tests/golden/lk_win_edges/lk_win_edges.npz
(the windows of k_lk_win in WIN_WINDOWS): LK starts that sit on the decision edges of calcOpticalFlowPyrLK's level-solve.

    python tests/golden/make_lk_edges.py                  W = 21 -> lk_edges.npz (about a minute on 8 cores)
    python tests/golden/make_lk_edges.py --windows        W = 4, 13, 16, 32 -> lk_win_edges.npz
    python tests/golden/make_lk_edges.py --win 21 --out F  W = 21 into F (to compare with lk_edges.npz)

Both are deterministic.

The images come from synth (recipes below, a SHA-256 of each image is stored); only the points and cv2's outputs are
stored.  A point is run through the reference's four-call ring L0->R0->R1->L1->L0 (call 0 is also the single call
L0->R0 of the GPU tests), the oracle's event log (oracle/lk_ref.c) tags the edges it reaches, and per category the
points closest to the edge are kept:
  MINEIG   level-0 minEig within 8 float ulps of 0.001f, both outcomes, 0.001f itself and the float below it
           (contrast-reduced images, then a sub-pixel grid search around the closest starts)
  HALF     |dx + pdx| or |dy + pdy| of an iteration j > 0 close to 0.01f, on both sides
  EPS      ||delta||^2 of an iteration close to eps^2 = 1e-4, on both sides
  CAP      the 30th iteration reached with its ||delta||^2 just above eps^2
  JOUT0 / JOUTC   the J window leaving the image mid-solve at level 0 / at a coarser level
  FINAL    the level-0 final re-check clearing the status
Points are tagged with every category they reach; tests/test_oracle_lk_edges.py and tests/test_oracle_lk_win_edges.py
re-derive the tags and margins.

At the windows of k_lk_win (which has no exact-integer path: every bit of b is the order of its float chains) the mining
also keeps, per wrong summation rule of the oracle (RULES, oracle/cref.py SUM_*) that applies at the window (APPLIES),
CAUGHT starts of the full-contrast recipe whose ring the rule changes.  The three window classes: W < 8 has no SIMD body
(nsimd = (W / 8) * 8 = 0, every column in the tail chain), W % 8 == 0 has no tail, any other W has both.  A rule that
reorders the lane reduction or the SIMD chains (SEQ, PAIRS, SCALAR, ADJ, COMBINE) needs a SIMD body; a column-major tail
(TAILCOL) needs a tail of two columns or more; a 4-wide split (SIMD4) moves columns only where W % 8 >= 4.  Elsewhere the
rule is the pinned computation, and changes nothing.  SEQ and PAIRS reorder the oracle's four-lane reductions, which
reach A only (b's lanes hold c0 + c2 and c1 + c3 by then); COMBINE is the (c0 + c1) + (c2 + c3) order for A and b alike.
"""
import hashlib
import json
import os
import sys
from multiprocessing import Pool

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle import cref                     # noqa: E402
from visual_odom_b200 import synth          # noqa: E402

# in directories of their own: tests/test_golden.py reads every tests/golden/*.npz as a ring golden vector
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "lk_edges", "lk_edges.npz")
WIN_OUT = os.path.join(HERE, "lk_win_edges", "lk_win_edges.npz")
# one window per class of k_lk_win (all-tail, SIMD + tail, no tail) and the largest, which reads the last padded column
WIN_WINDOWS = (4, 13, 16, 32)
RECIPES = [dict(w=1241, h=376, seed=5, scene="v1", contrast=1.0),
           dict(w=1241, h=376, seed=5, scene="v1", contrast=0.08)]
TAGS = ("MINEIG", "HALF", "EPS", "CAP", "JOUT0", "JOUTC", "FINAL")
BIT = {t: 1 << i for i, t in enumerate(TAGS)}
EPS2 = 1e-4
THR = np.float32(1e-3)
HALF_F = np.float32(0.01)
RING = ((0, 1), (1, 3), (3, 2), (2, 0))     # image indices (l0, r0, l1, r1) of the four calls
# wrong summation rules (oracle/cref.py) and the windows at which each one changes the computation
RULES = dict(SEQ=cref.SUM_SEQ, PAIRS=cref.SUM_PAIRS, SCALAR=cref.SUM_SCALAR, TAILCOL=cref.SUM_TAILCOL,
             SIMD4=cref.SUM_SIMD4, ADJ=cref.SUM_ADJ, COMBINE=cref.SUM_COMBINE)
CAUGHT = 3


def window_class(win):
    nsimd = (win // 8) * 8
    return "all-tail" if nsimd == 0 else "no-tail" if nsimd == win else "simd+tail"


def applies(rule, win):
    """does the wrong rule `rule` (a RULES key) compute anything differently at window `win`?"""
    nsimd = (win // 8) * 8
    if rule == "TAILCOL":
        return win - nsimd >= 2
    if rule == "SIMD4":
        return (win & ~3) != nsimd
    return nsimd > 0


# the applicability matrix at the mined windows, as written out (tests/test_oracle_lk_win_edges.py checks it against
# applies() and against the oracle)
APPLIES = {4: ("TAILCOL", "SIMD4"),
           13: ("SEQ", "PAIRS", "SCALAR", "TAILCOL", "SIMD4", "ADJ", "COMBINE"),
           16: ("SEQ", "PAIRS", "SCALAR", "ADJ", "COMBINE"),
           32: ("SEQ", "PAIRS", "SCALAR", "ADJ", "COMBINE")}


def images(r):
    """l0, r0, l1, r1 of a recipe: synth.stereo_unit, contrast scaled about 128 and rounded to u8."""
    u = synth.stereo_unit(r["w"], r["h"], r["seed"], scene=r["scene"])
    c = r["contrast"]
    return [np.clip(np.rint(128 + c * (u[k].astype(np.float64) - 128)), 0, 255).astype(np.uint8)
            for k in ("l0", "r0", "l1", "r1")]


def sha(img):
    return hashlib.sha256(np.ascontiguousarray(img).tobytes()).hexdigest()


def ulps(x, ref):
    """signed distance in float32 ulps of |x| from ref (both positive, same binade)"""
    return np.abs(np.asarray(x, np.float32)).view(np.int32).astype(np.int64) - int(np.float32(ref).view(np.int32))


def ring_oracle(imgs, pts, log=True, win=21):
    """The four chained calls on the oracle: [(out, status, err, log)] per call."""
    res, cur = [], np.ascontiguousarray(pts, np.float32)
    for a, b in RING:
        r = cref.lk_track(imgs[a], imgs[b], cur, win=win, return_log=log)
        res.append(r)
        cur = r[0]
    return res


def ring_cv2(imgs, pts, win=21):
    import cv2
    crit = (cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, 30, 0.01)
    outs, sts, errs, cur = [], [], [], np.ascontiguousarray(pts, np.float32)
    for a, b in RING:
        o, s, e = cv2.calcOpticalFlowPyrLK(imgs[a], imgs[b], cur.reshape(-1, 1, 2), None, winSize=(win, win), maxLevel=3,
                                           criteria=crit, flags=0, minEigThreshold=0.001)
        cur = o.reshape(-1, 2)
        outs.append(cur); sts.append(s.ravel()); errs.append(e.ravel())
    return np.stack(outs), np.stack(sts), np.stack(errs)


ITER_KINDS = (cref.EV_ITER, cref.EV_EPS, cref.EV_HALF, cref.EV_CAP)


def margins(log):
    """Per event of one call's log: the margin of each category (np.inf where it does not apply).  MINEIG, HALF in float
    ulps, EPS / CAP relative; JOUT0 / JOUTC / FINAL are 0 where the event happened."""
    n = len(log)
    m = {t: np.full(n, np.inf) for t in TAGS}
    k = log["kind"]
    st = ((k == cref.EV_SETUP) | (k == cref.EV_REJECT)) & (log["level"] == 0)
    m["MINEIG"][st] = np.abs(ulps(log["min_eig"][st], THR))
    it = np.isin(k, ITER_KINDS)
    j = it & (log["iter"] > 0)
    hx = np.abs(ulps(log["sdx"], HALF_F)).astype(np.float64)
    hy = np.abs(ulps(log["sdy"], HALF_F)).astype(np.float64)
    m["HALF"][j] = np.minimum(hx, hy)[j]
    m["EPS"][it] = np.abs(log["d2"][it] / EPS2 - 1)
    cap = k == cref.EV_CAP
    m["CAP"][cap] = np.where(log["d2"][cap] > EPS2, log["d2"][cap] / EPS2 - 1, np.inf)
    m["JOUT0"][(k == cref.EV_JOUT) & (log["level"] == 0)] = 0
    m["JOUTC"][(k == cref.EV_JOUT) & (log["level"] > 0)] = 0
    m["FINAL"][k == cref.EV_FINAL] = 0
    return m


def point_margins(logs, n):
    """Per point: the smallest margin of each category over the ring's four calls."""
    out = {t: np.full(n, np.inf) for t in TAGS}
    for log in logs:
        m = margins(log)
        for t in TAGS:
            np.minimum.at(out[t], log["pt"], m[t])
    return out


# category -> the margin under which a point counts
WITHIN = dict(MINEIG=8, HALF=64, EPS=1e-6, CAP=1e-2, JOUT0=0, JOUTC=0, FINAL=0)


def ring_changed(imgs, pts, mode, ref, win=21):
    """Per point: does the oracle under sum mode `mode` change any position or status of the ring against ref (the
    ring_oracle result in the pinned mode)?"""
    cref.lib().lk_set_sum_mode(mode)
    try:
        res = ring_oracle(imgs, pts, log=False, win=win)
    finally:
        cref.lib().lk_set_sum_mode(cref.SUM_CV2)
    bad = np.zeros(len(pts), bool)
    for r, rr in zip(res, ref):
        bad |= (r[0] != rr[0]).any(1) | (r[1] != rr[1])
    return bad


def _mine_main(args):
    """Random starts on the full-contrast recipe: FAST corners jittered by up to 1 px, and uniform starts over and
    around the image.  Returns (pts, margins) of the starts that reach any category."""
    seed, n, win = args
    imgs = images(RECIPES[0])
    w, h = RECIPES[0]["w"], RECIPES[0]["h"]
    rng = np.random.default_rng(seed)
    corners, _ = cref.fast_detect(imgs[0])
    a = corners[rng.integers(0, len(corners), n // 2)] + rng.uniform(-1, 1, (n // 2, 2))
    b = np.stack([rng.uniform(-40, w + 40, n - n // 2), rng.uniform(-40, h + 40, n - n // 2)], 1)
    pts = np.concatenate([a, b]).astype(np.float32)
    logs = [r[3] for r in ring_oracle(imgs, pts, win=win)]
    m = point_margins(logs, len(pts))
    keep = np.zeros(len(pts), bool)
    for t in TAGS:
        keep |= m[t] <= max(WITHIN[t], 1e-4 if t == "EPS" else WITHIN[t])
    return pts[keep], {t: m[t][keep] for t in TAGS}


def _min_eig0(img0, pts, win):
    """level-0 minEig of each start (one cheap single-level call)"""
    _, _, _, log = cref.lk_track(img0, img0, pts, win=win, max_level=0, max_count=1, return_log=True)
    st = log[(log["kind"] == cref.EV_SETUP) | (log["kind"] == cref.EV_REJECT)]
    me = np.full(len(pts), np.nan, np.float32)
    me[st["pt"]] = st["min_eig"]
    return me


def _mine_min_eig(args):
    """Contrast-reduced recipe: the closest of 100 k uniform starts, then a 64 x 64 grid of 2^-11 px around each."""
    seed, win = args
    imgs = images(RECIPES[1])
    w, h = RECIPES[1]["w"], RECIPES[1]["h"]
    rng = np.random.default_rng(seed)
    pts = np.stack([rng.uniform(0, w, 100000), rng.uniform(0, h, 100000)], 1).astype(np.float32)
    me = _min_eig0(imgs[0], pts, win)
    d = np.abs(me / np.float32(1e-3) - 1)
    best = pts[np.argsort(np.nan_to_num(d, nan=np.inf))[:12]]
    g = (np.arange(64) - 32) * 2.0 ** -11
    found = []
    for p in best:
        P = (p[None, None, :] + np.stack(np.meshgrid(g, g), -1)).reshape(-1, 2).astype(np.float32)
        u = ulps(_min_eig0(imgs[0], P, win), THR)
        ok = np.abs(u) <= 8
        found += [(q, int(v)) for q, v in zip(P[ok], u[ok])]
    return found


def _changed(args):
    """ring_changed on the full-contrast recipe (one chunk of starts)"""
    pts, mode, win = args
    imgs = images(RECIPES[0])
    return ring_changed(imgs, pts, mode, ring_oracle(imgs, pts, log=False, win=win), win)


def _catch_starts(pool, win):
    """Per wrong rule that applies at `win`, the first CAUGHT of 4000 FAST corners of the full-contrast recipe (jittered
    by up to 1 px) whose ring the rule changes."""
    imgs = images(RECIPES[0])
    corners, _ = cref.fast_detect(imgs[0])
    rng = np.random.default_rng(7000 + win)
    cand = (corners[rng.integers(0, len(corners), 4000)] + rng.uniform(-1, 1, (4000, 2))).astype(np.float32)
    chunks = np.array_split(cand, 8)
    out = []
    for rule in RULES:
        if not applies(rule, win):
            continue
        bad = np.concatenate(pool.map(_changed, [(c, RULES[rule], win) for c in chunks]))
        assert bad.sum() >= CAUGHT, (win, rule)
        out.append(cand[np.nonzero(bad)[0][:CAUGHT]])
    return np.concatenate(out)


def mine(pool, win, catches=False):
    """The fixture's arrays at one window: {name: array} with names as in lk_edges.npz (pts_0, out_0, ...)."""
    main_parts = pool.map(_mine_main, [(s, 20000, win) for s in range(16)])
    eig_parts = pool.map(_mine_min_eig, [(s, win) for s in range(4)])

    # ---- recipe 0: per category the points closest to the edge --------------------------------------------------
    pts0 = np.concatenate([p for p, _ in main_parts])
    m0 = {t: np.concatenate([m[t] for _, m in main_parts]) for t in TAGS}
    quota = dict(HALF=12, EPS=8, CAP=8, JOUT0=8, JOUTC=8, FINAL=8)
    sel = set()
    for t, q in quota.items():
        order = np.argsort(m0[t], kind="stable")
        sel.update(int(i) for i in order[:q] if np.isfinite(m0[t][i]))
    pts0 = pts0[sorted(sel)]
    if catches:
        pts0 = np.concatenate([pts0, _catch_starts(pool, win)])

    # ---- recipe 1: minEig around 0.001f -------------------------------------------------------------------------
    found = [f for part in eig_parts for f in part]
    by_ulp = {}
    for q, v in found:
        by_ulp.setdefault(v, []).append(q)
    pick = []
    for v in sorted(by_ulp):            # two starts per ulp value (the first two found), every value from -8 to 8
        pick += by_ulp[v][:2]
    pts1 = np.array(pick, np.float32).reshape(-1, 2)

    data = {}
    for ri, pts in enumerate((pts0, pts1)):
        imgs = images(RECIPES[ri])
        res = ring_oracle(imgs, pts, win=win)
        m = point_margins([r[3] for r in res], len(pts))
        tags = np.zeros(len(pts), np.int32)
        for t in TAGS:
            tags[m[t] <= WITHIN[t]] |= BIT[t]
        o, s, e = ring_cv2(imgs, pts, win)
        for k in range(4):
            assert np.array_equal(s[k], res[k][1]) and np.array_equal(o[k], res[k][0])
        data[f"sha256_{ri}"] = json.dumps([sha(a) for a in imgs])
        data[f"pts_{ri}"] = pts
        data[f"tags_{ri}"] = tags
        data[f"out_{ri}"] = o
        data[f"status_{ri}"] = s
        data[f"err_{ri}"] = np.where(s == 1, e, 0).astype(np.float32)
        print(f"W={win} recipe {ri}: {len(pts)} points;", ", ".join(f"{t} {int(((tags & BIT[t]) != 0).sum())} "
                                                                f"(best {m[t].min():.3g})" for t in TAGS))
    return data


def win_key(name, win):
    """lk_win_edges.npz's name of a per-window array: pts_0 at W = 13 is w13_pts_0 (the image hashes are shared)"""
    return name if name.startswith("sha256_") else f"w{win}_{name}"


def main():
    import argparse
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--windows", action="store_true", help=f"mine W = {WIN_WINDOWS} into {WIN_OUT}")
    ap.add_argument("--win", type=int, default=21, help="the window of a single-window fixture (default 21)")
    ap.add_argument("--out", help="where the fixture goes (default: its place under tests/golden)")
    args = ap.parse_args()
    base = dict(recipes=json.dumps(RECIPES), tags=json.dumps(TAGS))
    with Pool(min(8, os.cpu_count() or 1)) as pool:
        if args.windows:
            out = args.out or WIN_OUT
            data = dict(base, windows=json.dumps(WIN_WINDOWS), rules=json.dumps(list(RULES)))
            for win in WIN_WINDOWS:
                for k, v in mine(pool, win, catches=True).items():
                    data[win_key(k, win)] = v
        else:
            out = args.out or (OUT if args.win == 21 else None)
            assert out, "--out is needed at a window other than 21"
            data = dict(base, **mine(pool, args.win))
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    np.savez_compressed(out, **data)
    print(out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
