"""trackingFrame2Frame's mono_rotation branch per unit of the batched mode (vo_batch_mono_rotation, vo_batch_wait_mono,
vo_batch_fetch_mono, vo_batch_outputs_mono).

Units are KITTI-size synthetic stereo pairs with 2000 selected features; every configuration gets a fresh context.  The
expectation of every unit comes from one context that never switches the branch on: its records and point lists, and
vo_mono_rotation run on its filtered L0 / L1 lists with focal / pp = the float entries of P_l widened to double.  A unit
with the branch on must give that single-problem result bit for bit (status, counts, R, mask), carry its R in the record,
and leave every other record field and every list byte-identical to the branch off.
"""
import ctypes as C

import numpy as np
import pytest

from visual_odom_b200 import synth
from visual_odom_b200.capi import VO_E_TOO_FEW_POINTS, VO_OK, VoError

pytestmark = pytest.mark.gpu

W, H, B = 1241, 376, 8
N_SEL = 2000
T_PREV = (0.0, 0.0, -0.8)
ON = [1, 1, 0, 1, 1, 1, 0, 1]
LISTS = ("l0", "r0", "l1", "r1", "kept_idx", "X", "inliers")
PNP_FIELDS = ("n_features", "n_detected", "n_tracked", "n_valid", "n_inliers", "ransac_iters", "pnp_status", "rvec", "tvec")
P_L, P_R = synth.proj_matrices(synth.KITTI00)


def _context(**opts):
    from visual_odom_b200.capi import Context
    c = Context(0, max_features=2048)
    for k, v in opts.items():
        c.set_option(k, v)
    return c


def _configure(c, n=B):
    c.batch_configure(W, H, n, P_L, P_R)


def _dicts(us, pts=None):
    return [dict(u, t_prev=T_PREV, **({"pts": pts[i]} if pts is not None else {"n_select": N_SEL})) for i, u in enumerate(us)]


def _single(c, l0, l1, P_l):
    """vo_mono_rotation on one unit's lists: (rc, R, mask, n_inliers, iters)."""
    a = np.ascontiguousarray(l0, np.float32); b = np.ascontiguousarray(l1, np.float32)
    R = np.zeros(9); mask = np.zeros(max(len(a), 1), np.uint8); ni = C.c_int(0); it = C.c_int(0)
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    rc = c.lib.vo_mono_rotation(c.h, p(a), p(b), len(a), float(np.float32(P_l[0, 0])), float(np.float32(P_l[0, 2])),
                                float(np.float32(P_l[1, 2])), p(R), p(mask), C.byref(ni), C.byref(it))
    return rc, R.reshape(3, 3), mask[:len(a)].astype(bool), ni.value, it.value


def _expect_mono(c, base_rec, base_lists, P_l):
    rc, R, mask, ni, it = _single(c, base_lists["l0"], base_lists["l1"], P_l)
    if base_rec["n_valid"] < 5:
        rc = VO_E_TOO_FEW_POINTS            # vo_mono_rotation refuses n < 5 before it runs
    return dict(status=VO_OK if rc == VO_OK else VO_E_TOO_FEW_POINTS, R=R if rc == VO_OK else np.eye(3), mask=mask,
                n_inliers=ni, iters=it)


@pytest.fixture(scope="module")
def pool(built):
    """The units, and what a context without the branch gives for them (records, lists, single-problem mono results)."""
    us = [synth.stereo_unit(W, H, 300 + i, cal=synth.KITTI00) for i in range(B)]
    c = _context(batch_streams=1)
    _configure(c)
    arr, keep, pitch = c.make_units(_dicts(us))
    recs = c.frame_batch(arr, pitch)
    lists = [c.batch_fetch(i, recs[i]) for i in range(B)]
    mono = [_expect_mono(c, recs[i], lists[i], P_L) for i in range(B)]
    return dict(units=us, recs=recs, lists=lists, mono=mono)


def _same_pnp(got, base, where):
    for k in PNP_FIELDS:
        assert np.array_equal(np.asarray(got[k]), np.asarray(base[k])), (where, k)


def _check_mono(m, mask, exp, where):
    assert m["status"] == exp["status"], where
    assert np.array_equal(m["R"], exp["R"]), where
    if exp["status"] == VO_OK:
        assert m["n_inliers"] == exp["n_inliers"] and m["ransac_iters"] == exp["iters"], where
        assert np.array_equal(mask, exp["mask"]), where
        assert m["n_good"] > 0, where


def _check_unit(c, u, rec, base_rec, base_lists, exp, on, where, mono=None, outputs=False):
    """Record, lists, fetch_mono (and wait_mono's `mono`, outputs / outputs_mono) of unit u against the branch-off run."""
    _same_pnp(rec, base_rec, where)
    got = c.batch_fetch(u, rec)
    for k in LISTS:
        assert np.array_equal(got[k], base_lists[k]), (where, k)
    f = c.batch_fetch_mono(u, rec)
    if on:
        _check_mono(f["mono"], f["ess_mask"], exp, where)
        assert np.array_equal(rec["R"], f["mono"]["R"]), where
    else:
        assert f["mono"]["status"] == 0 and not f["mono"]["R"].any(), where
        assert np.array_equal(rec["R"], base_rec["R"]), where
    if mono is not None:
        for k in ("status", "n_inliers", "ransac_iters", "n_good", "R", "t"):
            assert np.array_equal(np.asarray(mono[k]), np.asarray(f["mono"][k])), (where, k)
    if outputs:
        o = c.batch_outputs(u, rec)
        for k in LISTS:
            assert np.array_equal(o[k], base_lists[k]), (where, "outputs", k)
        om = c.batch_outputs_mono(u, rec)
        for k in ("status", "n_inliers", "ransac_iters", "n_good", "R", "t"):
            assert np.array_equal(np.asarray(om["mono"][k]), np.asarray(f["mono"][k])), (where, "outputs_mono", k)
        if on:
            assert np.array_equal(om["ess_mask"], f["ess_mask"]), where


def _torch_units(us):
    import torch
    return [dict({k: torch.from_numpy(u[k]).cuda() for k in ("l0", "r0", "l1", "r1")}, n_select=N_SEL, t_prev=T_PREV) for u in us]


RANGES = [(0, 3), (3, 3), (6, 2)]
PATHS = [
    ("frame", dict(batch_streams=1)),
    ("frame", dict(batch_streams=2)),
    ("frame", dict(batch_streams=1, graphs=0)),
    ("upload", dict(batch_streams=2)),
    ("submit", dict(batch_outputs=1)),
    ("submit", dict(batch_outputs=0, graphs=0)),
    ("submit", dict(batch_outputs=1, sm_partition=0)),
    ("submit", dict(batch_outputs=1, sm_partition=8)),
    ("device", dict(batch_outputs=1)),
    ("rerun", dict(batch_outputs=1)),
]


@pytest.mark.parametrize("path,opts", PATHS, ids=[f"{p}-" + "-".join(f"{k}{v}" for k, v in o.items()) for p, o in PATHS])
def test_every_entry_path_gives_the_single_problem_bits(pool, path, opts):
    c = _context(**opts)
    _configure(c)
    c.batch_mono_rotation(0, ON)
    us = pool["units"]
    outputs = bool(opts.get("batch_outputs"))
    monos = [None] * B
    if path in ("frame", "upload"):
        arr, keep, pitch = c.make_units(_dicts(us))
        if path == "frame":
            recs = c.frame_batch(arr, pitch)
        else:
            c.batch_upload(arr, pitch); c.batch_run(); recs = c.batch_download(B)
    else:
        recs = [None] * B
        rounds = 2 if path == "rerun" else 1
        for r in range(rounds):
            keeps = []
            for u0, n in RANGES:            # three submissions in flight on disjoint slots
                if path == "device":
                    dev = _torch_units(us[u0:u0 + n])
                    keeps.append(dev)
                    c.batch_submit_device(dev, u0)
                elif r == 0:
                    arr, keep, pitch = c.make_units(_dicts(us[u0:u0 + n]))
                    keeps.append(keep)
                    c.batch_submit(arr, u0, pitch)
                else:
                    c.batch_submit(None, u0, pitch, n_units=n)
            for k, (u0, n) in enumerate(RANGES):
                if k == 2:
                    recs[u0:u0 + n] = c.batch_wait(u0, n)       # vo_batch_wait works too: R is the mono rotation
                else:
                    rs, ms = c.batch_wait_mono(u0, n)
                    recs[u0:u0 + n] = rs; monos[u0:u0 + n] = ms
    for u in range(B):
        _check_unit(c, u, recs[u], pool["recs"][u], pool["lists"][u], pool["mono"][u], ON[u], f"{path} unit {u}",
                    mono=monos[u], outputs=outputs and path not in ("frame", "upload"))


def test_against_cv2(pool):
    cv2 = pytest.importorskip("cv2")
    c = _context(batch_streams=1)
    _configure(c)
    c.batch_mono_rotation(0, [1] * B)
    arr, keep, pitch = c.make_units(_dicts(pool["units"]))
    recs = c.frame_batch(arr, pitch)
    for u in (0, 3, 7):
        l = pool["lists"][u]
        focal = float(P_L[0, 0]); pp = (float(P_L[0, 2]), float(P_L[1, 2]))
        E, mask = cv2.findEssentialMat(l["l0"], l["l1"], focal, pp, cv2.RANSAC, 0.999, 1.0)
        n_good, R, t, _ = cv2.recoverPose(E, l["l0"], l["l1"], focal=focal, pp=pp, mask=mask.copy())
        f = c.batch_fetch_mono(u, recs[u])
        assert f["mono"]["status"] == VO_OK
        assert np.array_equal(f["ess_mask"], mask.ravel().astype(bool)), u
        assert np.abs(f["mono"]["R"] - R).max() <= 1e-8, u
        assert np.abs(recs[u]["R"] - R).max() <= 1e-8, u
        assert f["mono"]["n_good"] == int(n_good), u


def test_mixed_ranges_match_each_unit_alone(pool):
    """Per-unit calibrations, parameters and switches in one range: each unit as in a context where it runs alone."""
    us = pool["units"][:4]
    scale = [1.0, 0.97, 1.03, 1.0]
    P_ls, P_rs = [], []
    for s in scale:
        cal = dict(synth.KITTI00, fx=synth.KITTI00["fx"] * s, fy=synth.KITTI00["fy"] * s, cx=synth.KITTI00["cx"] + 3 * (s - 1) * 100)
        a, b = synth.proj_matrices(cal)
        P_ls.append(a); P_rs.append(b)
    params = [None, dict(fast_threshold=15), dict(pnp_iterations=200), dict(circ_threshold=1)]
    on = [1, 0, 1, 1]
    c = _context(batch_streams=1)
    c.batch_configure(W, H, 4, P_ls[0], P_rs[0])
    c.batch_calibrate(0, np.array(P_ls), np.array(P_rs))
    c.batch_params(0, params)
    c.batch_mono_rotation(0, on)
    arr, keep, pitch = c.make_units(_dicts(us))
    recs = c.frame_batch(arr, pitch)
    for i in range(4):
        a = _context(batch_streams=1)
        a.batch_configure(W, H, 1, P_ls[i], P_rs[i])
        a.batch_params(0, [params[i]])
        a.batch_mono_rotation(0, [on[i]])
        arr1, keep1, pitch1 = a.make_units(_dicts(us[i:i + 1]))
        alone = a.frame_batch(arr1, pitch1)[0]
        for k in PNP_FIELDS + ("R",):
            assert np.array_equal(np.asarray(recs[i][k]), np.asarray(alone[k])), (i, k)
        got, ref = c.batch_fetch(i, recs[i]), a.batch_fetch(0, alone)
        for k in LISTS:
            assert np.array_equal(got[k], ref[k]), (i, k)
        fm, am = c.batch_fetch_mono(i, recs[i]), a.batch_fetch_mono(0, alone)
        for k in ("status", "n_inliers", "ransac_iters", "n_good", "R", "t"):
            assert np.array_equal(np.asarray(fm["mono"][k]), np.asarray(am["mono"][k])), (i, k)
        assert np.array_equal(fm["ess_mask"], am["ess_mask"]), i
        if on[i]:
            exp = _expect_mono(a, alone, ref, P_ls[i])
            _check_mono(fm["mono"], fm["ess_mask"], exp, i)


def test_toggling_inside_a_range_that_stays_on(pool):
    """The switch is read from device memory: toggles between runs of a range that keeps a unit on follow at once, on the
    captured graph of the context's stream and on pipelined submissions, at the same launch count."""
    us = pool["units"]
    patterns = [[1, 0, 0, 0, 0, 0, 0, 0], [0, 1, 1, 0, 0, 0, 0, 1], [1, 1, 1, 1, 1, 1, 1, 1], [1, 0, 0, 0, 0, 0, 0, 0]]
    c = _context(batch_streams=1, batch_outputs=1)
    _configure(c)
    arr, keep, pitch = c.make_units(_dicts(us))
    deltas = []
    for on in patterns:
        c.batch_mono_rotation(0, on)
        l0 = c.kernel_launches()
        recs = c.frame_batch(arr, pitch)
        deltas.append(c.kernel_launches() - l0)
        for u in range(B):
            _check_unit(c, u, recs[u], pool["recs"][u], pool["lists"][u], pool["mono"][u], on[u], f"frame {on} unit {u}")
        l0 = c.kernel_launches()
        c.batch_submit(None, 0, pitch, n_units=B)
        recs, ms = c.batch_wait_mono(0, B)
        deltas.append(c.kernel_launches() - l0)
        for u in range(B):
            _check_unit(c, u, recs[u], pool["recs"][u], pool["lists"][u], pool["mono"][u], on[u], f"submit {on} unit {u}",
                        mono=ms[u], outputs=True)
    assert len(set(deltas[0::2])) == 1 and len(set(deltas[1::2])) == 1, deltas


def test_abort_cases(pool):
    """Given feature lists: a unit with n_valid < 5, one with exactly 5 and one with more, in one range."""
    base = pool["lists"]
    full = [base[i]["pts_in"] for i in range(4)]
    pts = [full[0][base[0]["kept_idx"][:3]], full[1][base[1]["kept_idx"][:5]], full[2], full[3]]
    c = _context(batch_streams=1)
    _configure(c, 4)
    c.batch_mono_rotation(0, [1, 1, 1, 0])
    arr, keep, pitch = c.make_units(_dicts(pool["units"][:4], pts=pts))
    recs = c.frame_batch(arr, pitch)
    assert recs[0]["n_valid"] < 5 and recs[1]["n_valid"] == 5 and recs[2]["n_valid"] > 5, [r["n_valid"] for r in recs]
    for u in range(3):
        got = c.batch_fetch(u, recs[u])
        exp = _expect_mono(c, recs[u], got, P_L)
        f = c.batch_fetch_mono(u, recs[u])
        _check_mono(f["mono"], f["ess_mask"], exp, u)
        assert np.array_equal(recs[u]["R"], f["mono"]["R"]), u
        if exp["status"] != VO_OK:
            assert f["mono"]["status"] == VO_E_TOO_FEW_POINTS and np.array_equal(recs[u]["R"], np.eye(3)), u
    assert pool["mono"][2]["status"] == VO_OK
    # the neighbours of the aborting units: the same bits as with their full lists in the pool (given features: no
    # FAST corners counted)
    for u in (2, 3):
        for k in PNP_FIELDS:
            if k != "n_detected":
                assert np.array_equal(np.asarray(recs[u][k]), np.asarray(pool["recs"][u][k])), (u, k)
    _check_mono(c.batch_fetch_mono(2, recs[2])["mono"], c.batch_fetch_mono(2, recs[2])["ess_mask"], pool["mono"][2], 2)
    assert np.array_equal(recs[3]["R"], pool["recs"][3]["R"])


def _submit_launches(c, us, on):
    _configure(c)
    if on is not None:
        c.batch_mono_rotation(0, on)
    arr, keep, pitch = c.make_units(_dicts(us))
    out = []
    for _ in range(2):
        l0 = c.kernel_launches()
        c.batch_submit(arr, 0, pitch)
        c.batch_wait(0, B)
        out.append(c.kernel_launches() - l0)
    assert out[0] == out[1]
    return out[0]


def test_launches(pool):
    us = pool["units"]
    never = _submit_launches(_context(), us, None)
    off = _submit_launches(_context(), us, [0] * B)
    one = _submit_launches(_context(), us, [0, 0, 0, 1, 0, 0, 0, 0])
    all_on = _submit_launches(_context(), us, [1] * B)
    assert off == never
    assert one == all_on and one > never, (never, one, all_on)


def test_refusals_change_nothing(pool):
    us = pool["units"]
    c = _context(batch_outputs=0)
    _configure(c)
    c.batch_mono_rotation(0, ON)
    with pytest.raises(VoError):
        c.batch_mono_rotation(6, [1, 1, 1])                  # past the configured units
    with pytest.raises(VoError):
        c.batch_mono_rotation(-1, [1])
    arr, keep, pitch = c.make_units(_dicts(us))
    c.batch_submit(arr, 0, pitch)
    with pytest.raises(VoError):
        c.batch_mono_rotation(0, [0] * B)                    # a submission in flight
    with pytest.raises(VoError):
        c.batch_fetch_mono(0, pool["recs"][0])               # not waited for
    recs, ms = c.batch_wait_mono(0, B)
    with pytest.raises(VoError):
        c.batch_outputs_mono(0, recs[0])                     # batch_outputs is off
    for u in range(B):                                       # the switches are those set before the refusals
        _check_unit(c, u, recs[u], pool["recs"][u], pool["lists"][u], pool["mono"][u], ON[u], f"unit {u}", mono=ms[u])
    # vo_batch_configure switches every unit off
    _configure(c)
    recs = c.frame_batch(arr, pitch)
    for u in range(B):
        _check_unit(c, u, recs[u], pool["recs"][u], pool["lists"][u], pool["mono"][u], 0, f"reconfigured unit {u}")
