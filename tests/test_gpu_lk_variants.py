"""The LK ring kernel under every work schedule the library can launch, bit for bit against the oracle (oracle/lk_ref.c,
pinned to cv2 in test_oracle_lk.py).

The default launch is what test_gpu_lk.py sees.  Here every configuration gets a fresh context and runs the same inputs:
work items of 1, 2, 3, 5, 7 phases (lk_span): the running estimate and the progress counter are handed from item to
item, items straddle call boundaries, and an item may end mid-call.
The automatic span only applies to a launch with more features than resident warps; the tests check that their inputs
are that large on the GPU they run on.  Consecutive configurations alternate between two input sets, so a
launch that skipped work cannot pass on what the previous context left in recycled device memory.
"""
import numpy as np
import pytest

from visual_odom_b200 import synth

pytestmark = pytest.mark.gpu

W, H = 1241, 376
N_FAST = 6000
SPANS = (0, 1, 2, 3, 5, 7, 16)         # 0 = automatic
LK_WARPS_PER_CTA = 2                   # visual_odom_b200/csrc/lk_ring.h
LK_CTAS_PER_SM = 8


def _border_points(w, h):
    return np.array([[0, 0], [-5, 3], [w - 1, h - 1], [w + 5, 10], [3, h + 30], [-30, -30], [w - 0.5, 5.5],
                     [10.25, -21.5], [w + 20.9, h / 2], [5, -10.99], [-11.01, 7]], np.float32)


def _inputs(seed):
    """A KITTI-size unit with a flat patch on all four images and FAST-selected + border + scattered points, and a
    100x44 unit (a two-level pyramid: a ring of 8 phases) with points scattered over and around it."""
    from oracle import cref
    rng = np.random.default_rng(seed)
    u = synth.stereo_unit(W, H, seed, scene="v1")
    imgs = [u[k].copy() for k in ("l0", "r0", "l1", "r1")]
    for a in imgs:
        a[H // 3: H // 3 + 40, W // 4: W // 4 + 60] = 128            # minEig < 1e-3: rejected at every level
    # 4 levels: a single call has 4 phases (span 3 ends an item at level 1, the next starts mid-call), a ring 16
    assert cref.Pyramid(imgs[0]).nlevels() == 4
    corners, _ = cref.fast_detect(imgs[0])
    feats = synth.select_features(corners, N_FAST)
    assert len(feats) == N_FAST
    scattered = np.stack([rng.uniform(-60, W + 60, 1200), rng.uniform(-60, H + 60, 1200)], 1).astype(np.float32)
    scattered[:50] = np.round(scattered[:50])                         # integer positions (zero fractional weights)
    pts = np.concatenate([feats, _border_points(W, H), scattered])
    s = synth.stereo_unit(100, 44, seed + 100, scene="v0")
    assert cref.Pyramid(s["l0"]).nlevels() == 2
    spts = np.stack([rng.uniform(-10, 110, 4000), rng.uniform(-10, 54, 4000)], 1).astype(np.float32)
    return dict(imgs=imgs, pts=pts, small=[s[k] for k in ("l0", "r0", "l1", "r1")], small_pts=spts)


def _ring_ref(imgs, pts):
    from oracle import ref_path
    fs = ref_path.FeatureSet()
    fs.points = pts.copy(); fs.ages = np.arange(len(pts), dtype=np.int32) % 7
    ages0 = fs.ages.copy()
    ref = ref_path.circular_matching(*imgs, pts, fs, backend="c")
    return dict(ref=ref, ages0=ages0, ages=fs.ages.copy())


@pytest.fixture(scope="module")
def cases(built):
    """Two input sets and their oracle results, computed once for every configuration."""
    from oracle import cref
    out = []
    for seed in (21, 22):
        x = _inputs(seed)
        x["single_ref"] = cref.lk_track(x["imgs"][0], x["imgs"][2], x["pts"])        # L0 -> L1: not a call of the ring
        x["ring_ref"] = _ring_ref(x["imgs"], x["pts"])
        x["small_ref"] = _ring_ref(x["small"], x["small_pts"])
        out.append(x)
    return out


def _check_ring(got, r):
    ref = r["ref"]
    assert np.array_equal(got["status4"], ref["raw"]["status"]), "ring status differs"
    for k, name in enumerate(("r0", "r1", "l1", "l0_ret")):
        bad = np.nonzero((got["raw4"][k] != ref["raw"][name]).any(1))[0]
        assert len(bad) == 0, f"raw {name} differs at {len(bad)} points, first {bad[:8]}"
    assert np.array_equal(got["kept_idx"], ref["kept_idx"])
    for name in ("l0", "r0", "l1", "r1", "l0_ret"):
        assert np.array_equal(got[name], ref[name]), name
    assert np.array_equal(got["ages"], r["ages"])


def _run(case, opts, need_big):
    """Single call, ring + filters on the KITTI-size unit and ring on the small unit, on a fresh context with `opts`."""
    import torch
    from visual_odom_b200.capi import Context
    c = Context(0, max_features=8192)
    try:
        for k, v in opts.items():
            c.set_option(k, v)
        resident_warps = torch.cuda.get_device_properties(0).multi_processor_count * LK_CTAS_PER_SM * LK_WARPS_PER_CTA
        if need_big:            # the automatic span only applies above the resident warps
            assert len(case["pts"]) > resident_warps, (len(case["pts"]), resident_warps)
        ro, rs, re = case["single_ref"]
        go, gs, ge = c.lk_track(case["imgs"][0], case["imgs"][2], case["pts"])
        assert np.array_equal(gs, rs), f"status differs at {np.nonzero(gs != rs)[0][:8]}"
        bad = np.nonzero((go != ro).any(1))[0]
        assert len(bad) == 0, f"single call: positions differ at {len(bad)} points, first {bad[:8]}"
        assert np.array_equal(ge[rs == 1], re[rs == 1])
        assert 0.5 * len(rs) < rs.sum() < len(rs)
        _check_ring(c.circular_match(*case["imgs"], case["pts"], ages=case["ring_ref"]["ages0"]), case["ring_ref"])
        _check_ring(c.circular_match(*case["small"], case["small_pts"], ages=case["small_ref"]["ages0"]), case["small_ref"])
    finally:
        c.close()


CONFIGS = [dict(lk_span=s) for s in SPANS]


@pytest.mark.parametrize("i", range(len(CONFIGS)),
                         ids=["-".join(f"{k}={v}" for k, v in cfg.items()) for cfg in CONFIGS])
def test_lk_variant_bit_exact(cases, i):
    cfg = CONFIGS[i]
    _run(cases[i % 2], cfg, need_big=cfg["lk_span"] == 0)
