"""Batched results into device memory (vo_batch_wait_device).

Every case runs on a fresh context and compares, bit for bit, against a twin context fed the same calls but retired
through the host: vo_batch_wait (records), vo_batch_fetch (pts4, kept_idx, points3D, inliers), vo_batch_wait_mono and
vo_batch_fetch_mono (mono results, essential masks).  Units are KITTI-size synthetic stereo pairs with 2000 features, as
in the benchmark, with detected or given features, per-unit calibrations and parameters, from gray or BGR device images
and from units == NULL re-runs.  Also covered: three submissions in flight retired out of order with host and device
waits mixed, a range resubmitted right after each device wait (the pinned input staging), the non-blocking return and a
consumer on the same stream, the calls behind the shared-buffer gate right after a device wait, the record gather, the
refusals and the launch counts.
"""
import ctypes as C
import time

import numpy as np
import pytest

from visual_odom_b200 import capi, synth
from visual_odom_b200.capi import RESULT_DTYPE, VO_E_INVALID, VoBatchDResults, VoError

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

W, H, B = 1241, 376, 8
N_SEL = 2000
T_PREV = (0.0, 0.0, -0.8)
IMGS = ("l0", "r0", "l1", "r1")
NAMES4 = ("l0", "r0", "l1", "r1")
RANGES = [(0, 3), (3, 3), (6, 2)]
P_L, P_R = synth.proj_matrices(synth.KITTI00)
SENTINEL = 0xA5


def _context(**opts):
    c = capi.Context(0, max_features=2048)
    for k, v in opts.items():
        c.set_option(k, v)
    c.batch_configure(W, H, B, P_L, P_R)
    return c


@pytest.fixture(scope="module")
def pool(built):
    """The units (host arrays and CUDA copies) and the features a detection run selects for them."""
    us = [synth.stereo_unit(W, H, 500 + i, cal=synth.KITTI00) for i in range(B)]
    c = _context(batch_streams=1)
    arr, keep, pitch = c.make_units([dict(u, n_select=N_SEL, t_prev=T_PREV) for u in us])
    recs = c.frame_batch(arr, pitch)
    pts = [c.batch_fetch(i, recs[i])["pts_in"].copy() for i in range(B)]
    c.close()
    gray = [{k: torch.from_numpy(u[k]).cuda() for k in IMGS} for u in us]
    bgr = [{k: g[k].unsqueeze(-1).expand(-1, -1, 3).contiguous() for k in IMGS} for g in gray]
    return dict(units=us, gray=gray, bgr=bgr, pts=pts)


def _dunits(pool, u0, n, colour=False, pts=None, t_prev=T_PREV):
    """batch_submit_device units for slots [u0, u0 + n): pool units u0 .., detected features unless `pts` (a list per unit)."""
    src = pool["bgr" if colour else "gray"]
    out = []
    for i in range(n):
        d = dict(src[u0 + i], t_prev=t_prev[i] if isinstance(t_prev, list) else t_prev)
        if colour:
            d["order"] = "bgr"
        if pts is None:
            d["n_select"] = N_SEL
        else:
            d["pts"] = pts[i]
        out.append(d)
    return out


def _host_results(c, u0, n, mono=False):
    """The twin's retirement of [u0, u0 + n): raw records, each unit's lists (and mono results / masks)."""
    if mono:                                                 # the C call itself, so the records keep their padding bytes
        res, ms = (capi.VoUnitResult * n)(), (capi.VoMonoResult * n)()
        c._check(c.lib.vo_batch_wait_mono(c.h, u0, n, res, ms))
        raw = np.frombuffer(bytes(res), dtype=RESULT_DTYPE)
        ms = [bytes(m) for m in ms]
    else:
        raw = c.batch_wait(u0, n, raw=True)
        ms = None
    recs = c.records_to_dicts(raw)
    lists = [c.batch_fetch(u0 + i, recs[i]) for i in range(n)]
    fm = [c.batch_fetch_mono(u0 + i, recs[i]) for i in range(n)] if mono else None
    return dict(raw=raw, recs=recs, lists=lists, mono=ms, fetch_mono=fm)


def _snapshot(out):
    """A stream-ordered copy of the tensors a device wait filled (a consumer on the same stream, no synchronise)."""
    return {k: v.clone() for k, v in out.items() if isinstance(v, torch.Tensor) and k in
            ("records", "pts4", "kept_idx", "points3d", "inliers", "mono_raw", "ess_mask")}


def _np(snap):
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in snap.items()}


def _same(dev, ref, cap, where, sentinel=False):
    """Device results (numpy) against the twin's: records byte for byte, the first min(n, cap) list entries byte for byte
    (and, with sentinel, every byte past them still the sentinel)."""
    n = len(ref["raw"])
    assert dev["records"].tobytes() == ref["raw"].tobytes(), where
    for i, r in enumerate(ref["recs"]):
        nv, ni = min(r["n_valid"], cap), min(r["n_inliers"], cap)
        L = ref["lists"][i]
        parts = []
        if "pts4" in dev:
            for k, name in enumerate(NAMES4):
                parts.append((f"pts4[{name}]", dev["pts4"][i, k], np.ascontiguousarray(L[name], np.float32), nv))
        if "kept_idx" in dev:
            parts.append(("kept_idx", dev["kept_idx"][i], L["kept_idx"], nv))
        if "points3d" in dev:
            parts.append(("points3d", dev["points3d"][i], L["X"], nv))
        if "inliers" in dev:
            parts.append(("inliers", dev["inliers"][i], L["inliers"], ni))
        for name, got, want, m in parts:
            assert got[:m].tobytes() == np.ascontiguousarray(want[:m]).astype(got.dtype).tobytes(), (where, i, name, m)
            if sentinel:
                rest = got[m:].view(np.uint8)
                assert (rest == SENTINEL).all(), (where, i, name, "written past", m)
    assert n == dev["records"].shape[0]


def _fill(out):
    for k in ("pts4", "kept_idx", "points3d", "inliers", "ess_mask", "mono_raw"):
        if k in out:
            out[k].view(torch.uint8).fill_(SENTINEL)


# ---- the device wait against the host wait -------------------------------------------------------------------------
CASES = [
    ("gray", "detect", dict()),
    ("gray", "given", dict()),
    ("bgr", "detect", dict(graphs=0)),
    ("bgr", "given", dict(sm_partition=0)),
    ("gray", "calib", dict(sm_partition=8)),
    ("rerun", "detect", dict(graphs=1, sm_partition=0)),
    ("rerun", "given", dict(graphs=0, sm_partition=8)),
]


def _setup_calib(c):
    """Per-unit calibrations and parameters on every unit."""
    P_ls, P_rs = [], []
    for u in range(B):
        s = 1.0 + 0.01 * (u - 3)
        a, b = synth.proj_matrices(dict(synth.KITTI00, fx=synth.KITTI00["fx"] * s, fy=synth.KITTI00["fy"] * s))
        P_ls.append(a); P_rs.append(b)
    c.batch_calibrate(0, np.array(P_ls), np.array(P_rs))
    c.batch_params(0, [None, dict(fast_threshold=15), dict(pnp_iterations=200), dict(circ_threshold=1), None,
                       dict(pnp_reproj_error=2.0), dict(lk_max_iters=20), None])


@pytest.mark.parametrize("inputs,features,opts", CASES, ids=[f"{i}-{f}-" + "-".join(f"{k}{v}" for k, v in o.items()) for i, f, o in CASES])
def test_device_wait_matches_the_host_wait(pool, inputs, features, opts):
    a, b = _context(**opts), _context(**opts)
    if features == "calib":
        _setup_calib(a); _setup_calib(b)
    pts = pool["pts"] if features == "given" else None
    for c in (a, b):
        for u0, n in RANGES:                                 # three submissions in flight on disjoint slot ranges
            c.batch_submit_device(_dunits(pool, u0, n, inputs == "bgr", None if pts is None else pts[u0:u0 + n]), u0)
    if inputs == "rerun":                                    # retire through the host, then re-run what is resident
        for c in (a, b):
            for u0, n in RANGES:
                c.batch_wait(u0, n)
            for u0, n in RANGES:
                c.batch_submit_device(None, u0, n_units=n)
    snaps = {}
    for u0, n in RANGES:
        snaps[u0] = _snapshot(a.batch_wait_device(u0, n, pts_cap=2048))
    for u0, n in RANGES:
        _same(_np(snaps[u0]), _host_results(b, u0, n), 2048, f"{inputs}/{features} [{u0}, {u0 + n})")
    a.close(); b.close()


def test_out_of_order_retirement_mixing_host_and_device_waits(pool):
    a, b = _context(), _context()
    for c in (a, b):
        for u0, n in RANGES:
            c.batch_submit_device(_dunits(pool, u0, n), u0)
    snap2 = _snapshot(a.batch_wait_device(6, 2))             # the last submission first, on the device
    raw0 = a.batch_wait(0, 3, raw=True)                      # the first through the host
    snap1 = _snapshot(a.batch_wait_device(3, 3))
    ref = {u0: _host_results(b, u0, n) for u0, n in RANGES[::-1]}
    _same(_np(snap2), ref[6], 2048, "range 6 (device, first)")
    _same(_np(snap1), ref[3], 2048, "range 3 (device, last)")
    assert raw0.tobytes() == ref[0]["raw"].tobytes()
    recs0 = a.records_to_dicts(raw0)
    for i in range(3):
        got = a.batch_fetch(i, recs0[i])
        for k in NAMES4 + ("kept_idx", "X", "inliers"):
            assert got[k].tobytes() == ref[0]["lists"][i][k].tobytes(), (i, k)
    # and the device-waited units read back the same through the blocking calls
    for i in range(2):
        got = a.batch_fetch(6 + i, ref[6]["recs"][i])
        for k in NAMES4 + ("kept_idx", "X", "inliers"):
            assert got[k].tobytes() == ref[6]["lists"][i][k].tobytes(), (6 + i, k)
    a.close(); b.close()


def test_resubmitting_a_range_right_after_each_device_wait(pool):
    """Different t_prev, feature lists and counts every step: a submission that read the previous step's pinned staging
    (t_prev, counts, image descriptors) would give different bits."""
    a, b = _context(), _context()
    n, steps = 4, 8
    out = a.batch_dresults_alloc(n, pts_cap=2048)
    seen, want = [], []
    rng = np.random.default_rng(5)
    plan = []
    for s in range(steps):
        u0 = 4 * (s % 2)                                     # the two halves swap images so the descriptors differ too
        pts = [pool["pts"][(u0 + i + s) % B][: N_SEL - 150 * ((i + s) % 5)] for i in range(n)]
        tp = [(float(rng.normal(0, 0.05)), 0.0, float(-0.8 + 0.1 * rng.normal())) for _ in range(n)]
        plan.append((u0, pts, tp))
    for s, (u0, pts, tp) in enumerate(plan):
        a.batch_submit_device(_dunits(pool, u0, n, pts=pts, t_prev=tp), 0)
        a.batch_wait_device(0, n, out=out)
        seen.append(_snapshot(out))                          # consumer on the stream, before the next wait overwrites out
    for s, (u0, pts, tp) in enumerate(plan):
        b.batch_submit_device(_dunits(pool, u0, n, pts=pts, t_prev=tp), 0)
        want.append(_host_results(b, 0, n))
    for s in range(steps):
        _same(_np(seen[s]), want[s], 2048, f"step {s}")
    assert len({r["tvec"][2] for w in want for r in w["recs"]}) > n       # the steps really differ
    a.close(); b.close()


def test_mono_with_mixed_switches(pool):
    on = [1, 0, 1, 1, 0, 0, 1, 0]
    a, b = _context(batch_outputs=1), _context(batch_outputs=1)
    for c in (a, b):
        c.batch_mono_rotation(0, on)
        c.batch_submit_device(_dunits(pool, 0, B), 0)
    out = a.batch_dresults_alloc(B, pts_cap=2048, mono=True)
    _fill(out)
    a.batch_wait_device(0, B, out=out)
    dev = _np(_snapshot(out))
    ref = _host_results(b, 0, B, mono=True)
    _same(dev, ref, 2048, "mono", sentinel=True)
    m = dev["mono_raw"]
    for u in range(B):
        assert m[u].tobytes() == ref["mono"][u], u           # vo_batch_wait_mono's bytes (zeroed for a unit that is off)
        if not on[u]:
            assert not m[u].view(np.uint8).any(), u
            assert (dev["ess_mask"][u] == SENTINEL).all(), u     # untouched
            continue
        fm = ref["fetch_mono"][u]
        assert m[u, 2:11].tobytes() == np.ascontiguousarray(fm["mono"]["R"], np.float64).tobytes(), u
        assert ref["recs"][u]["R"].tobytes() == np.ascontiguousarray(fm["mono"]["R"], np.float64).tobytes(), u
        nv = ref["recs"][u]["n_valid"]
        assert np.array_equal(dev["ess_mask"][u, :nv].astype(bool), fm["ess_mask"]), u
        assert (dev["ess_mask"][u, nv:] == SENTINEL).all(), u
    a.close(); b.close()


def test_a_small_pts_cap_writes_exactly_its_entries(pool):
    cap = 600
    a, b = _context(), _context()
    for c in (a, b):
        c.batch_submit_device(_dunits(pool, 0, B), 0)
    out = a.batch_dresults_alloc(B, pts_cap=cap)
    _fill(out)
    a.batch_wait_device(0, B, out=out)
    ref = _host_results(b, 0, B)
    assert any(r["n_valid"] > cap for r in ref["recs"])
    _same(_np(_snapshot(out)), ref, cap, f"pts_cap {cap}", sentinel=True)
    a.close(); b.close()


def test_consumer_after_the_call_and_no_host_wait(pool):
    a, b = _context(), _context()
    out = a.batch_dresults_alloc(B, pts_cap=2048)
    seen, busy, want = [], [], []
    tps = [[(0.0, 0.0, -0.8 - 0.05 * s)] * B for s in range(4)]
    for s in range(4):
        torch.cuda._sleep(200_000_000)                       # ~0.1 s of GPU time ahead of the submission
        a.batch_submit_device(_dunits(pool, 0, B, t_prev=tps[s]), 0)
        t0 = time.perf_counter()
        a.batch_wait_device(0, B, out=out)
        dt = time.perf_counter() - t0
        busy.append((not torch.cuda.current_stream().query(), dt))
        seen.append(_snapshot(out))
    for s in range(4):
        b.batch_submit_device(_dunits(pool, 0, B, t_prev=tps[s]), 0)
        want.append(_host_results(b, 0, B))
    for s in range(4):
        _same(_np(seen[s]), want[s], 2048, f"step {s}")
    assert all(x for x, _ in busy), busy
    assert all(dt < 0.05 for _, dt in busy), busy
    a.close(); b.close()


# ---- the shared-buffer gate right after a device wait --------------------------------------------------------------
def _other_calibration():
    return synth.proj_matrices(dict(synth.KITTI00, fx=synth.KITTI00["fx"] * 1.05, fy=synth.KITTI00["fy"] * 1.05))


GATE = {
    "calibrate": lambda c, pool: c.batch_calibrate(0, np.array([_other_calibration()[0]] * B), np.array([_other_calibration()[1]] * B)),
    "params": lambda c, pool: c.batch_params(0, [dict(fast_threshold=15, pnp_iterations=50)] * B),
    "mono_rotation": lambda c, pool: c.batch_mono_rotation(0, [1] * B),
    "configure": lambda c, pool: c.batch_configure(W, H, B, *_other_calibration()),
    "seq_begin": lambda c, pool: c.seq_begin(pool["units"][0]["l0"], pool["units"][0]["r0"], P_L, P_R),
}


@pytest.mark.parametrize("call", list(GATE) + ["outputs", "fetch"])
def test_calls_right_after_a_device_wait(pool, call):
    a, b = _context(batch_outputs=1), _context(batch_outputs=1)
    for c in (a, b):
        c.batch_submit_device(_dunits(pool, 0, B), 0)
    snap = _snapshot(a.batch_wait_device(0, B, pts_cap=2048))
    ref = _host_results(b, 0, B)
    if call in GATE:
        GATE[call](a, pool)                                  # changes what the retired submission read, had it not finished
        _same(_np(snap), ref, 2048, call)
        if call != "seq_begin":                              # the next submission follows the new settings like the twin's
            GATE[call](b, pool)
            for c in (a, b):
                c.batch_submit_device(_dunits(pool, 0, B), 0)
            snap2 = _snapshot(a.batch_wait_device(0, B, pts_cap=2048))
            _same(_np(snap2), _host_results(b, 0, B), 2048, call + " then a submission")
    else:
        for u in range(B):
            got = a.batch_outputs(u, ref["recs"][u]) if call == "outputs" else a.batch_fetch(u, ref["recs"][u])
            for k in NAMES4 + ("kept_idx", "X", "inliers"):
                assert got[k].tobytes() == ref["lists"][u][k].tobytes(), (call, u, k)
        _same(_np(snap), ref, 2048, call)
    a.close(); b.close()


def test_record_gather_after_device_waits(pool):
    a = _context()
    try:
        try:
            uid = a.dist_unique_id()
        except RuntimeError:
            pytest.skip("no loadable NCCL on this host")
        a.dist_init(uid, 0, 1)
        snaps = []
        for s in range(3):
            a.batch_submit_device(_dunits(pool, 0, 4, t_prev=(0.0, 0.0, -0.8 - 0.1 * s)), 0)
            snaps.append(_snapshot(a.batch_wait_device(0, 4, points=False, kept_idx=False, points3d=False, inliers=False)))
            a.dist_gather_post(0, 4)
        recs = [_np(s)["records"] for s in snaps]
        assert len({r.tobytes() for r in recs}) == 3
        for s in range(3):
            got = a.dist_gather_wait(4, raw=True)
            assert got.tobytes() == recs[s].tobytes(), s
    finally:
        a.close()


# ---- refusals and launch counts ------------------------------------------------------------------------------------
def test_refusals_leave_the_submission_pending(pool):
    a, b = _context(), _context()
    arr, keep, pitch = a.make_units([dict(u, n_select=N_SEL, t_prev=T_PREV) for u in pool["units"]])
    out = a.batch_dresults_alloc(B, pts_cap=2048)

    def refused(fn, match):
        with pytest.raises(VoError, match=match) as e:
            fn()
        assert e.value.code == VO_E_INVALID, str(e.value)

    def raw_call(r):
        a._enter_stream()
        return a.lib.vo_batch_wait_device(a.h, 0, B, None if r is None else C.byref(r))

    def table(**kw):
        r = VoBatchDResults()
        r.records, r.pts_cap = out["records"].data_ptr(), 2048
        for k, v in kw.items():
            setattr(r, k, v)
        return r

    # a host-image submission: refused, then vo_batch_wait returns it
    a.batch_submit(arr, 0, pitch)
    b.batch_submit(arr, 0, pitch)
    refused(lambda: a.batch_wait_device(0, B, out=out), "host images")
    ref = _host_results(b, 0, B)
    assert a.batch_wait(0, B, raw=True).tobytes() == ref["raw"].tobytes()
    # a device submission: every refusal below changes nothing
    for c in (a, b):
        c.batch_submit_device(_dunits(pool, 0, B), 0)
    refused(lambda: a.batch_wait_device(0, 4), "no pending")
    refused(lambda: a.batch_wait_device(1, B - 1), "no pending")
    assert raw_call(None) == VO_E_INVALID
    assert raw_call(table(pts_cap=-1)) == VO_E_INVALID
    assert raw_call(table(pts_cap=0, pts4=out["pts4"].data_ptr())) == VO_E_INVALID
    host = np.zeros((B, 19))
    assert raw_call(table(records=host.ctypes.data)) == VO_E_INVALID
    pinned = torch.zeros((B, 2048), dtype=torch.int32).pin_memory()
    assert raw_call(table(inliers=pinned.data_ptr())) == VO_E_INVALID
    assert "device memory" in a.lib.vo_last_error(a.h).decode()
    torch.cuda.synchronize()
    assert not out["records"].any()                          # nothing written
    ref = _host_results(b, 0, B)
    raw = a.batch_wait(0, B, raw=True)
    assert raw.tobytes() == ref["raw"].tobytes()
    recs = a.records_to_dicts(raw)
    for u in range(B):
        got = a.batch_fetch(u, recs[u])
        for k in NAMES4 + ("kept_idx", "X", "inliers"):
            assert got[k].tobytes() == ref["lists"][u][k].tobytes(), (u, k)
    a.close(); b.close()


def test_one_launch_per_device_wait(pool):
    a, b = _context(), _context()
    counts = {"device": [], "host": []}
    for c, kind in ((a, "device"), (b, "host")):
        for s in range(3):
            l0 = c.kernel_launches()
            c.batch_submit_device(_dunits(pool, 0, B), 0)
            l1 = c.kernel_launches()
            if kind == "device":
                c.batch_wait_device(0, B)
            else:
                c.batch_wait(0, B)
            counts[kind].append((l1 - l0, c.kernel_launches() - l1))
    assert all(w == 1 for _, w in counts["device"]), counts
    assert all(w == 0 for _, w in counts["host"]), counts
    assert [s for s, _ in counts["device"]] == [s for s, _ in counts["host"]], counts
    torch.cuda.synchronize()
    a.close(); b.close()
