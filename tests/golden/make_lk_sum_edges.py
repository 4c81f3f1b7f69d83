"""Mines tests/golden/lk_sum_edges/lk_sum_edges.npz: LK starts whose Newton iterations sit on the edges of k_lk_ring's
choice between its two ways of forming b1 / b2.

    python tests/golden/make_lk_sum_edges.py      (about a minute on 8 cores; deterministic)

The kernel sums the ten b chains (4 SIMD chains and a tail, for b1 and for b2) as integers and combines the chain totals
in float as tail + ((c0 + c2) + (c1 + c3)) when its vote passes: max(P, N) <= 2^24 on every chain, P and N the sums of
the chain's positive products and of the magnitudes of its negative ones, so that every prefix sum is an exact float.
Otherwise it replays cv2's float chains, and does so for the rest of the level-solve.  An iteration the kernel votes on
is one with no rejected iteration before it in its level-solve.  Categories, from the oracle's event log
(oracle/lk_ref.c, per chain P, N, the total and cv2's float chain):
  VOTE_IN    voted, accepted, with the largest max(P, N) just below (or at) 2^24, half of them on a b1 chain and half on
             a b2 chain; margin 2^24 - max(P, N)
  VOTE_OUT   voted, rejected, with the largest max(P, N) just above 2^24 and a float chain that differs from its integer
             total rounded to float: a vote twice as permissive takes the exact path there and gets b wrong;
             margin max(P, N) - 2^24
  TAIL_ONLY  voted, rejected only because of a tail chain, whose float chain differs from its integer total
  B2_ONLY    voted, rejected only because of a b2 chain, whose float chain differs from its integer total
  COMBINE    voted, accepted, and (c0 + c1) + (c2 + c3) gives another b1 or b2 than cv2's (c0 + c2) + (c1 + c3)
The images come from synth (recipes below, a SHA-256 of each image is stored); only the points and cv2's outputs are
stored.  A point is run through the reference's four-call ring L0->R0->R1->L1->L0 (call 0 is also the single call L0->R0
of the GPU tests) and tagged with every category it reaches in any call.  FAST corners jittered by up to 1 px give the
candidates; a 32 x 32 grid of 2^-10 px around the closest VOTE_IN and VOTE_OUT starts pushes those margins down.
"""
import json
import os
import sys
from multiprocessing import Pool

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)
from oracle import cref                     # noqa: E402
import make_lk_edges as mk                  # noqa: E402  (images, sha, ring_oracle, ring_cv2)

# in a directory of its own: tests/test_golden.py reads every tests/golden/*.npz as a ring golden vector
OUT = os.path.join(HERE, "lk_sum_edges", "lk_sum_edges.npz")
# the benchmark scene, and a half-contrast scene on which most iterations pass the vote
RECIPES = [dict(w=1241, h=376, seed=0, scene="v1", contrast=1.0),
           dict(w=1241, h=376, seed=5, scene="v1", contrast=0.5)]
TAGS = ("VOTE_IN", "VOTE_OUT", "TAIL_ONLY", "B2_ONLY", "COMBINE")
BIT = {t: 1 << i for i, t in enumerate(TAGS)}
LIM = 1 << 24
ITER_KINDS = (cref.EV_ITER, cref.EV_EPS, cref.EV_HALF, cref.EV_CAP)
SIMD = [0, 1, 2, 3, 5, 6, 7, 8]              # chain indices: b1 chains 0..3, b1 tail 4, b2 chains 5..8, b2 tail 9
TAIL = [4, 9]
# category -> the margin under which an iteration counts (VOTE_IN / VOTE_OUT in units of 2^24; the others are events)
WITHIN = dict(VOTE_IN=1e-4, VOTE_OUT=5e-2, TAIL_ONLY=0, B2_ONLY=0, COMBINE=0)
QUOTA = dict(VOTE_IN=8, VOTE_OUT=8, TAIL_ONLY=6, B2_ONLY=6, COMBINE=8)     # points kept per category and recipe
# A wrong rule changes b by an ulp or so on the iterations of its category, and that mostly vanishes once added to the
# position; so per wrong rule (oracle/cref.py SUM_M*) the category whose starts show it, and how many starts of that
# category whose ring the rule changes are kept besides the QUOTA
CATCHES = {cref.SUM_M1: "VOTE_OUT", cref.SUM_M2: "VOTE_OUT", cref.SUM_M3: "TAIL_ONLY", cref.SUM_M4: "B2_ONLY",
           cref.SUM_M5: "COMBINE", cref.SUM_M6: "TAIL_ONLY"}
CAUGHT = 3


def combine(c, order):
    """the exact path's float combination of chain totals c (float32, [..., 5]): tail + simd, simd in cv2's order
    (c0 + c2) + (c1 + c3) or in the order (c0 + c1) + (c2 + c3)"""
    if order == "cv2":
        s = (c[..., 0] + c[..., 2]) + (c[..., 1] + c[..., 3])
    else:
        s = (c[..., 0] + c[..., 1]) + (c[..., 2] + c[..., 3])
    return c[..., 4] + s


def iterations(log):
    """The Newton iterations of one call's log, with per iteration: pn (max(P, N) per chain), accept (the kernel's
    vote), voted (no rejected iteration before it in its level-solve) and fsame (per chain: cv2's float chain equals
    the integer total rounded to float)."""
    it = log[np.isin(log["kind"], ITER_KINDS)]
    pn = np.maximum(it["pos"], it["neg"])
    accept = (pn <= LIM).all(1)
    rej = (~accept).astype(np.int64)
    start = it["iter"] == 0                 # each level-solve's iterations begin with iteration 0
    gid = np.cumsum(start) - 1
    excl = np.cumsum(rej) - rej
    voted = excl - excl[np.nonzero(start)[0]][gid] == 0
    fsame = it["fchain"] == it["total"].astype(np.float32)
    return dict(it=it, pn=pn, accept=accept, voted=voted, fsame=fsame)


def margins(log):
    """Per Newton iteration of one call's log: (pt, the margin of each category (np.inf where it does not apply),
    the side of VOTE_IN's largest chain: 0 for b1, 1 for b2)."""
    t = iterations(log)
    it, pn, acc, vot, fs = t["it"], t["pn"], t["accept"], t["voted"], t["fsame"]
    n = len(it)
    m = {k: np.full(n, np.inf) for k in TAGS}
    top = pn.max(1)
    fits = pn <= LIM
    sel = vot & acc
    m["VOTE_IN"][sel] = (LIM - top[sel]) / LIM
    sel = vot & ~acc & (top <= 2 * LIM) & ~fs.all(1)
    m["VOTE_OUT"][sel] = (top[sel] - LIM) / LIM
    m["TAIL_ONLY"][vot & ~acc & fits[:, SIMD].all(1) & ~fs[:, TAIL].all(1)] = 0
    m["B2_ONLY"][vot & ~acc & fits[:, :5].all(1) & ~fs[:, 5:].all(1)] = 0
    c = it["total"].astype(np.float32)
    diff = np.zeros(n, bool)
    for q in (slice(0, 5), slice(5, 10)):
        diff |= combine(c[:, q], "cv2") != combine(c[:, q], "pairs")
    m["COMBINE"][vot & acc & diff] = 0
    side = (pn.argmax(1) >= 5).astype(np.int32)
    return it["pt"], m, side


def point_margins(logs, n):
    """Per point: the smallest margin of each category over the given calls, and VOTE_IN's side at that margin."""
    out = {t: np.full(n, np.inf) for t in TAGS}
    side = np.full(n, -1, np.int32)
    for log in logs:
        pt, m, sd = margins(log)
        for t in TAGS:
            np.minimum.at(out[t], pt, m[t])
        # the side of the iteration that sets the point's VOTE_IN margin
        o = np.lexsort((m["VOTE_IN"], pt))
        pt_o, m_o, sd_o = pt[o], m["VOTE_IN"][o], sd[o]
        first = np.r_[True, pt_o[1:] != pt_o[:-1]]
        hit = first & (m_o <= out["VOTE_IN"][pt_o])
        side[pt_o[hit]] = sd_o[hit]
    return out, side


def _random_starts(args):
    """FAST corners of l0 jittered by up to 1 px: (pts, margins, side) of the starts that reach any category."""
    ri, seed, n = args
    imgs = mk.images(RECIPES[ri])
    rng = np.random.default_rng(1000 * ri + seed)
    corners, _ = cref.fast_detect(imgs[0])
    pts = (corners[rng.integers(0, len(corners), n)] + rng.uniform(-1, 1, (n, 2))).astype(np.float32)
    m, side = point_margins([r[3] for r in mk.ring_oracle(imgs, pts)], n)
    keep = np.zeros(n, bool)
    for t in TAGS:
        keep |= np.isfinite(m[t])
    return pts[keep], {t: m[t][keep] for t in TAGS}, side[keep]


def _grid(args):
    """A 32 x 32 grid of 2^-10 px around a start, judged on call 0: (pts, margins, side) of the grid points that
    reach VOTE_IN or VOTE_OUT."""
    ri, p = args
    imgs = mk.images(RECIPES[ri])
    g = (np.arange(32) - 16) * 2.0 ** -10
    P = (p[None, None, :] + np.stack(np.meshgrid(g, g), -1)).reshape(-1, 2).astype(np.float32)
    log = cref.lk_track(imgs[0], imgs[1], P, return_log=True)[3]
    m, side = point_margins([log], len(P))
    keep = np.isfinite(m["VOTE_IN"]) | np.isfinite(m["VOTE_OUT"])
    return P[keep], {t: m[t][keep] for t in TAGS}, side[keep]


def _cat(parts):
    return (np.concatenate([p for p, _, _ in parts]),
            {t: np.concatenate([m[t] for _, m, _ in parts]) for t in TAGS},
            np.concatenate([s for _, _, s in parts]))


def ring_changed(imgs, pts, mode, ref):
    """Per point: does the oracle under sum mode `mode` change any position or status of the ring against ref (the
    ring_oracle result in the pinned mode)?"""
    cref.lib().lk_set_sum_mode(mode)
    try:
        res = mk.ring_oracle(imgs, pts, log=False)
    finally:
        cref.lib().lk_set_sum_mode(cref.SUM_CV2)
    bad = np.zeros(len(pts), bool)
    for r, rr in zip(res, ref):
        bad |= (r[0] != rr[0]).any(1) | (r[1] != rr[1])
    return bad


def _changed(args):
    ri, pts, mode = args
    imgs = mk.images(RECIPES[ri])
    return ring_changed(imgs, pts, mode, mk.ring_oracle(imgs, pts, log=False))


def select(pool, ri, pts, m, side):
    """Per category the QUOTA points closest to its edge (VOTE_IN: half with the b1 side, half with the b2 side), and
    per wrong sum rule the CAUGHT points of its category closest to the edge among those whose ring it changes."""
    sel = []
    for t, q in QUOTA.items():
        if t == "VOTE_IN":
            for sd in (0, 1):
                mm = np.where(side == sd, m[t], np.inf)
                sel += [int(i) for i in np.argsort(mm, kind="stable")[:q // 2] if np.isfinite(mm[i])]
        else:
            sel += [int(i) for i in np.argsort(m[t], kind="stable")[:q] if np.isfinite(m[t][i])]
    for mode, t in CATCHES.items():
        cand = [int(i) for i in np.argsort(m[t], kind="stable")[:400] if m[t][i] <= WITHIN[t]]
        chunks = np.array_split(np.array(cand, np.int64), 8)
        bad = np.concatenate(pool.map(_changed, [(ri, pts[c], mode) for c in chunks]))
        sel += [c for c, b in zip(cand, bad) if b][:CAUGHT]
    return pts[sorted(set(sel))]


def main():
    data = dict(recipes=json.dumps(RECIPES), tags=json.dumps(TAGS))
    with Pool(min(8, os.cpu_count() or 1)) as pool:
        for ri in range(len(RECIPES)):
            pts, m, side = _cat(pool.map(_random_starts, [(ri, s, 2000) for s in range(8)]))
            # grid search around the closest VOTE_IN starts of each side and the closest VOTE_OUT starts
            seeds = []
            for sd in (0, 1):
                mm = np.where(side == sd, m["VOTE_IN"], np.inf)
                seeds += [pts[i] for i in np.argsort(mm, kind="stable")[:4] if np.isfinite(mm[i])]
            seeds += [pts[i] for i in np.argsort(m["VOTE_OUT"], kind="stable")[:4] if np.isfinite(m["VOTE_OUT"][i])]
            gp, gm, gs = _cat(pool.map(_grid, [(ri, p) for p in seeds]))
            pts = select(pool, ri, np.concatenate([pts, gp]), {t: np.concatenate([m[t], gm[t]]) for t in TAGS},
                         np.concatenate([side, gs]))

            imgs = mk.images(RECIPES[ri])
            res = mk.ring_oracle(imgs, pts)
            pm, _ = point_margins([r[3] for r in res], len(pts))
            tags = np.zeros(len(pts), np.int32)
            for t in TAGS:
                tags[pm[t] <= WITHIN[t]] |= BIT[t]
            o, s, e = mk.ring_cv2(imgs, pts)
            for k in range(4):
                assert np.array_equal(s[k], res[k][1]) and np.array_equal(o[k], res[k][0])
            data[f"sha256_{ri}"] = json.dumps([mk.sha(a) for a in imgs])
            data[f"pts_{ri}"] = pts
            data[f"tags_{ri}"] = tags
            data[f"out_{ri}"] = o
            data[f"status_{ri}"] = s
            data[f"err_{ri}"] = np.where(s == 1, e, 0).astype(np.float32)
            print(f"recipe {ri}: {len(pts)} points;", ", ".join(
                f"{t} {int(((tags & BIT[t]) != 0).sum())} (best {pm[t].min() * (LIM if t.startswith('VOTE') else 1):.6g})"
                for t in TAGS))
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    np.savez_compressed(OUT, **data)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
