"""Multi-sequence runs that return their results into GPU memory (flag VO_MSEQ_DEVICE_RESULTS, vo_mseq_wait_device):
frame by frame and bit for bit, the statuses, records, point lists and frame_pose equal those of the same run waited on
the host (vo_mseq_wait), points3D equals vo_triangulate (and cv2), the inlier list equals vo_pnp_ransac (and the oracle),
starts and retirements report and reset as on the host, the device pose gate equals vo_pose_step across its boundary,
the wait neither blocks the host nor breaks the stream contract, refusals change nothing, and a wait is one launch.
Every case runs on a fresh context."""

import time

import numpy as np
import pytest

from visual_odom_b200 import capi, synth

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
cv2 = pytest.importorskip("cv2")

K0 = synth.KITTI00
INTS = ("n_features", "n_detected", "n_tracked", "n_valid", "n_inliers", "ransac_iters", "pnp_status")
NF = 5                      # frames per drive: the first pair and four submissions

def _cal(sx=1.0, dcx=0.0, dcy=0.0, sb=1.0):
    return dict(fx=K0["fx"] * sx, fy=K0["fy"] * sx, cx=K0["cx"] + dcx, cy=K0["cy"] + dcy, bf=K0["bf"] * sb)

_FRAMES = {}

def _drive(w, h, seed, cal=None, n=NF, steps=None):
    """(P_l, P_r, [(left, right) CUDA tensors] * n) of one synthetic drive; steps[k] = (rvec, tvec) of frame k."""
    cal = cal or _cal(1.0, (w - 1241) / 2.0, (h - 376) / 2.0)
    steps = steps or [(np.array((0.001, -0.004, 0.0005)) * k, np.array((0.01, -0.003, -0.2)) * k) for k in range(n)]
    key = (w, h, seed, tuple(sorted(cal.items())), tuple(tuple(np.r_[r, t]) for r, t in steps))
    if key not in _FRAMES:
        base = synth.stereo_unit(w, h, seed, cal=cal)
        fr = [(base["l0"], base["r0"])]
        for r, t in steps[1:]:
            u = synth.stereo_unit(w, h, seed, cal=cal, rvec=np.asarray(r), tvec=np.asarray(t))
            fr.append((u["l1"], u["r1"]))
        dev = [(torch.from_numpy(l).cuda(), torch.from_numpy(r).cuda()) for l, r in fr]
        _FRAMES[key] = (base["P_l"], base["P_r"], dev)
    return _FRAMES[key]

def _fresh(**kw):
    return capi.Context(0, max_features=8192, **kw)

def _mats(drives):
    return np.stack([d[0] for d in drives]), np.stack([d[1] for d in drives])

def _pair(drives, k):
    return [d[2][k][0] for d in drives], [d[2][k][1] for d in drives]

def _host_run(drives, mono=False, graphs=True):
    """The unflagged reference: device input, host waits, two submissions in flight; per submission (records, frame poses
    right after its wait)."""
    c = _fresh()
    c.set_option("graphs", int(graphs))
    n = len(drives)
    c.mseq_begin_device(*_pair(drives, 0), *_mats(drives), mono_rotation=mono)
    out = []
    c.mseq_submit_device(*_pair(drives, 1))
    for k in range(1, NF):
        if k + 1 < NF:
            c.mseq_submit_device(*_pair(drives, k + 1))
        recs = c.mseq_wait(mono=mono)
        out.append((recs, np.stack([c.mseq_pose(q) for q in range(n)])))
    c.close()
    return out

def _snap(out):
    """Host copies of one mseq_wait_device result (after a synchronise)."""
    return {k: v.cpu().numpy() for k, v in out.items() if isinstance(v, torch.Tensor)}

def _device_run(drives, mono=False, graphs=True, ctx=None, pts_cap=4096):
    """The flagged run, two submissions in flight, each result copied out after the run's end: per submission the
    host copies of the tensors mseq_wait_device filled (a fresh set per wait)."""
    c = ctx or _fresh()
    c.set_option("graphs", int(graphs))
    c.mseq_begin_device(*_pair(drives, 0), *_mats(drives), mono_rotation=mono, device_results=True)
    res = []
    c.mseq_submit_device(*_pair(drives, 1))
    for k in range(1, NF):
        if k + 1 < NF:
            c.mseq_submit_device(*_pair(drives, k + 1))
        res.append(c.mseq_wait_device(pts_cap=pts_cap))
    torch.cuda.synchronize()
    out = [_snap(r) for r in res]
    if ctx is None:
        c.close()
    return out

def _same(got, want, what):
    assert len(got) == len(want)
    for k, (g, (recs, poses)) in enumerate(zip(got, want)):
        for q, w in enumerate(recs):
            where = f"{what}: submission {k + 1} sequence {q}"
            assert g["status"][q] == w["status"], where
            for i, f in enumerate(INTS):
                assert g["counts"][q, i] == w[f], f"{where}: {f}"
            for f in ("rvec", "tvec", "R"):
                assert np.array_equal(g[f][q], w[f]), f"{where}: {f}"
            nv = w["n_valid"] if w["status"] in (capi.VO_OK, capi.VO_E_CAPACITY) else 0
            for i, f in enumerate(("l0", "r0", "l1", "r1")):
                assert np.array_equal(g["pts4"][q, i, :nv], w[f]), f"{where}: {f}"
            if "mono" in w:
                m = w["mono"]
                assert list(g["mono_counts"][q]) == [m["status"], m["n_inliers"], m["ransac_iters"], m["n_good"]], where
                assert np.array_equal(g["mono_R"][q], m["R"]) and np.array_equal(g["mono_t"][q], m["t"]), where
                assert np.array_equal(g["ess_mask"][q, :nv].astype(bool), w["ess_mask"]), f"{where}: ess_mask"
            if poses is not None:
                assert np.array_equal(g["frame_pose"][q], poses[q]), f"{where}: frame_pose"

DRIVES_5 = [(640, 240, 31), (640, 240, 7), (1241, 376, 11), (640, 240, 13), (1241, 376, 23)]

@pytest.mark.parametrize("n_seq", [1, 5])
def test_flagged_equals_unflagged(built, n_seq):
    drives = [_drive(*d) for d in DRIVES_5[:n_seq]]
    want = _host_run(drives)
    _same(_device_run(drives), want, f"n_seq={n_seq}")
    assert all(r["n_inliers"] > 20 for r in want[-1][0])

def test_kitti_sizes_and_cameras(built):
    drives = [_drive(1241, 376, 3, _cal()), _drive(1242, 375, 4, _cal(0.98, 0.5, -0.5, 1.02)),
              _drive(1226, 370, 6, _cal(1.01, -7.5, -3.0, 0.97))]
    _same(_device_run(drives), _host_run(drives), "kitti")

def test_graphs_off(built):
    drives = [_drive(640, 240, 31), _drive(1241, 376, 11)]
    _same(_device_run(drives, graphs=False), _host_run(drives), "graphs=0")

def test_mono_rotation(built):
    drives = [_drive(640, 240, 31), _drive(640, 240, 7), _drive(601, 233, 13)]
    want = _host_run(drives, mono=True)
    _same(_device_run(drives, mono=True), want, "mono")
    assert all(r["mono"]["status"] == 0 for r in want[-1][0])

# ---- points3D and inliers ------------------------------------------------------------------------------------------
def test_points3d_and_inliers_equal_the_stage_calls(built):
    from oracle import pnp_ref, ref_path
    drives = [_drive(640, 240, 31), _drive(1242, 375, 4, _cal(0.98, 0.5, -0.5, 1.02)), _drive(1241, 376, 11)]
    got = _device_run(drives)
    c = _fresh()
    t_prev = [np.zeros(3)] * len(drives)
    checked = 0
    for k, g in enumerate(got):
        for q, (P_l, P_r, _) in enumerate(drives):
            nv, ni = int(g["counts"][q, 3]), int(g["counts"][q, 4])
            l0, r0, l1 = g["pts4"][q, 0, :nv], g["pts4"][q, 1, :nv], g["pts4"][q, 2, :nv]
            X = g["points3d"][q, :nv]
            assert np.array_equal(X, c.triangulate(P_l, P_r, l0, r0)), f"submission {k + 1} sequence {q}: points3d"
            K = np.asarray(P_l, np.float32)[:, :3]
            ref = c.pnp_ransac(X, l1, K, tvec0=t_prev[q])
            assert len(ref["inliers"]) == ni and np.array_equal(g["inliers"][q, :ni], ref["inliers"]), \
                f"submission {k + 1} sequence {q}: inliers"
            assert np.array_equal(ref["tvec"], g["tvec"][q])
            if q == 0:          # one sequence against cv2 and the oracle's solvePnPRansac
                H = cv2.triangulatePoints(np.asarray(P_l, np.float32), np.asarray(P_r, np.float32), l0.T.copy(), r0.T.copy())
                assert np.array_equal(X, cv2.convertPointsFromHomogeneous(H.T).reshape(-1, 3)), "cv2 points3D"
                o = pnp_ref.solve_pnp_ransac(X, l1, K.astype(np.float64), np.zeros(3), t_prev[q], confidence=ref_path.PNP_CONFIDENCE)
                assert np.array_equal(g["inliers"][q, :ni], o["inliers"]), "oracle inliers"
            t_prev[q] = g["tvec"][q].copy()
            checked += ni
    c.close()
    assert checked > 1000

# ---- starts and retirements ----------------------------------------------------------------------------------------
ENV = (656, 248)
SLOT_DRIVES = {"a": (656, 248, 13), "b": (512, 200, 42), "c": (640, 240, 31), "d": (601, 233, 7), "e": (620, 236, 23)}
# slot 0: a drive retired at 4 and a smaller one started at 5 (into the slot the frame in flight retires); slot 1: a
# live drive replaced at 3; slot 2: an empty slot started at 2; slot 3: empty throughout
SCHED = [(0, 1, "a", 3), (0, 5, "b", 3), (1, 1, "c", 2), (1, 3, "d", 4), (2, 2, "e", 5)]
N_SLOTS, K_LAST = 4, 7

def _slot_run(flagged, mono=False):
    frames = {k: _drive(*v, n=5) for k, v in SLOT_DRIVES.items()}
    c = _fresh()
    c.mseq_open(N_SLOTS, *ENV, mono_rotation=mono, device_results=flagged)

    def go(k):
        lefts, rights, start = [None] * N_SLOTS, [None] * N_SLOTS, {}
        for q, k0, d, L in SCHED:
            if k0 <= k < k0 + L:
                lefts[q], rights[q] = frames[d][2][k - k0]
                if k == k0:
                    start[q] = frames[d][:2]
        c.mseq_submit_device(lefts, rights, start=start)
    out = []
    go(1)
    for k in range(1, K_LAST + 1):
        if k < K_LAST:
            go(k + 1)
        if flagged:
            out.append(c.mseq_wait_device())
        else:
            out.append((c.mseq_wait(mono=mono), np.stack([c.mseq_pose(q) for q in range(N_SLOTS)])))
    if flagged:
        torch.cuda.synchronize()
        out = [_snap(r) for r in out]
    poses = [c.mseq_pose(q) for q in range(N_SLOTS)]
    c.close()
    return out, poses

def test_starts_and_retirements(built):
    want, want_pose = _slot_run(False)
    got, got_pose = _slot_run(True)
    _same(got, want, "slots")
    st = [[r["status"] for r in recs] for recs, _ in want]
    assert st[0] == [capi.VO_MSEQ_STARTED, capi.VO_MSEQ_STARTED, capi.VO_MSEQ_RETIRED, capi.VO_MSEQ_RETIRED]
    assert st[1][2] == capi.VO_MSEQ_STARTED and st[2][1] == capi.VO_MSEQ_STARTED and st[4][0] == capi.VO_MSEQ_STARTED
    for g, s in zip(got, st):
        for q in range(N_SLOTS):
            if s[q] in (capi.VO_MSEQ_STARTED, capi.VO_MSEQ_RETIRED):
                assert not g["records"][q].any(), "a retired or started slot's record is zeroed"
            if s[q] == capi.VO_MSEQ_STARTED:
                assert np.array_equal(g["frame_pose"][q], np.eye(4)), "a start resets the pose"
    for a, b in zip(got_pose, want_pose):
        assert np.array_equal(a, b)

# ---- pose gates ----------------------------------------------------------------------------------------------------
def test_pose_gates_in_a_drive(built):
    """Frame 2 turns 0.12 rad beyond frame 1 (the Euler gate) and frame 4 repeats frame 3 (the 0.05 scale gate)."""
    r, t = np.array((0.001, -0.004, 0.0005)), np.array((0.01, -0.003, -0.2))
    steps = [(0 * r, 0 * t), (r, t), (r + (0.0, 0.12, 0.0), 2 * t), (3 * r, 3 * t), (3 * r, 3 * t)]
    drives = [_drive(640, 240, 31, steps=steps), _drive(1241, 376, 11, steps=steps)]
    want = _host_run(drives)
    _same(_device_run(drives), want, "gates")

def _rot(axis, a):
    c, s = np.cos(a), np.sin(a)
    R = np.eye(3)
    i, j = [(1, 2), (0, 2), (0, 1)][axis]
    R[i, i], R[i, j], R[j, i], R[j, j] = c, -s, s, c
    if axis == 1:
        R = R.T
    return R

def test_pose_step_device_equals_the_host_across_the_gate(built):
    """R swept in double ulps through the float midpoint of 0.099999994f / 0.1f on every axis, both signs, both sy
    branches, and random rotations: pose and return code equal vo_pose_step bit for bit."""
    m = (float(np.float32(0.1)) + float(np.nextafter(np.float32(0.1), np.float32(0)))) / 2
    Rs = []
    # entries that carry each angle: x: atan2(R7, R8), y: atan2(-R6, sy), z: atan2(R3, R0)
    for axis, idx in ((0, 7), (1, 6), (2, 3)):
        for sign in (1, -1):
            base = _rot(axis, sign * m).reshape(9)
            for k in range(-48, 49):
                R = base.copy()
                R[idx] = R[idx] + k * np.spacing(R[idx])
                Rs.append(R)
    # the sy < 1e-6 branch (R0 = 1e-7, R3 = 0; R6 = -1e-9 keeps y small and the matrix invertible): x from atan2(-R5, R4)
    for sign in (1, -1):
        for k in range(-48, 49):
            R = np.zeros(9)
            R[0], R[2], R[6], R[7] = 1e-7, 1.0, -1e-9, 1.0
            R[4], R[5] = np.cos(m), -sign * np.sin(m)
            R[5] += k * np.spacing(R[5])
            Rs.append(R)
    rng = np.random.default_rng(3)
    for _ in range(2000):
        a = rng.normal(0, 0.06, 3)
        Rs.append((_rot(0, a[0]) @ _rot(1, a[1]) @ _rot(2, a[2])).reshape(9))
    Rs = np.array(Rs)
    n = len(Rs)
    ts = np.tile([0.01, -0.003, -0.8], (n, 1))
    ts[::7] *= 0.01                                 # under the 0.05 scale gate
    pose0 = np.tile(np.eye(4), (n, 1, 1))
    pose0[:, :3, 3] = rng.normal(0, 5, (n, 3))
    want_p, want_rc = [], []
    lib = capi.load_library()
    for i in range(n):                              # vo_pose_step itself, its return code included
        p, R, t = pose0[i].copy(), np.ascontiguousarray(Rs[i]), np.ascontiguousarray(ts[i])
        want_rc.append(lib.vo_pose_step(capi._p(p), capi._p(R), capi._p(t)))
        want_p.append(p)
    c = _fresh()
    got_p, got_rc = c.pose_step_device(pose0, Rs.reshape(n, 3, 3), ts)
    c.close()
    assert np.array_equal(got_rc, want_rc)
    assert np.array_equal(got_p, np.array(want_p))
    sweep = np.array(want_rc[:6 * 97 + 2 * 97])
    assert 0 < sweep.sum() < len(sweep), "the sweep crosses the gate"

# ---- stream contract and non-blocking -------------------------------------------------------------------------------
def test_consumer_after_the_call_and_no_host_wait(built):
    drives = [_drive(640, 240, 31), _drive(1241, 376, 11)]
    want = _host_run(drives)
    c = _fresh()
    c.mseq_begin_device(*_pair(drives, 0), *_mats(drives), device_results=True)
    out = c.mseq_dresults_alloc()                   # one set of tensors, reused by every wait
    seen, returned_busy = [], []
    c.mseq_submit_device(*_pair(drives, 1))
    for k in range(1, NF):
        torch.cuda._sleep(200_000_000)              # ~0.1 s of GPU time ahead of the submission
        if k + 1 < NF:
            c.mseq_submit_device(*_pair(drives, k + 1))
        t0 = time.perf_counter()
        c.mseq_wait_device(out=out)
        dt = time.perf_counter() - t0
        returned_busy.append((not torch.cuda.current_stream().query(), dt))
        # a consumer on the same stream, no synchronise: it reads this wait's results before the next wait overwrites them
        seen.append({k2: v.clone() for k2, v in out.items() if isinstance(v, torch.Tensor)})
    torch.cuda.synchronize()
    _same([{k2: v.cpu().numpy() for k2, v in s.items()} for s in seen], want, "consumer")
    assert all(busy for busy, _ in returned_busy), returned_busy
    assert all(dt < 0.05 for _, dt in returned_busy), returned_busy
    c.close()

# ---- refusals ------------------------------------------------------------------------------------------------------
def test_refusals_change_nothing(built):
    drives = [_drive(640, 240, 31), _drive(601, 233, 7), _drive(640, 240, 13)]
    want = _host_run(drives)
    c = _fresh()

    def expect(fn, match):
        with pytest.raises(capi.VoError, match=match) as e:
            fn()
        assert e.value.code == capi.VO_E_INVALID, (e.value.code, str(e.value))
    host = [d[2][1][0].cpu().numpy() for d in drives]
    c.mseq_begin_device(*_pair(drives, 0), *_mats(drives), device_results=True)
    expect(lambda: c.mseq_wait_device(), "no frame in flight")
    res = []
    c.mseq_submit_device(*_pair(drives, 1))
    for k in range(1, NF):
        if k == 2:
            expect(lambda: c.mseq_submit(host, host), "vo_mseq_submit_device only")
            expect(lambda: c.mseq_wait(), "vo_mseq_wait_device")
            expect(lambda: c.mseq_wait(mono=True), "vo_mseq_wait_device")
            r = capi.VoMseqDResults()
            hp = np.zeros(3, np.int32)
            r.status = hp.ctypes.data
            expect(lambda: c._device_call(c.lib.vo_mseq_wait_device, C_byref(r)), "not device memory")
            m = torch.zeros((3, 14), dtype=torch.float64, device="cuda")
            r = capi.VoMseqDResults(); r.mono = m.data_ptr()
            expect(lambda: c._device_call(c.lib.vo_mseq_wait_device, C_byref(r)), "VO_MSEQ_MONO_ROTATION")
            p4 = torch.zeros((3, 4, 1, 2), dtype=torch.float32, device="cuda")
            r = capi.VoMseqDResults(); r.pts4 = p4.data_ptr(); r.pts_cap = 0
            expect(lambda: c._device_call(c.lib.vo_mseq_wait_device, C_byref(r)), "pts_cap")
        if k + 1 < NF:
            c.mseq_submit_device(*_pair(drives, k + 1))
        res.append(c.mseq_wait_device())
    torch.cuda.synchronize()
    _same([_snap(r) for r in res], want, "after refusals")
    # the unflagged run refuses the device wait
    c.mseq_begin_device(*_pair(drives, 0), *_mats(drives))
    c.mseq_submit_device(*_pair(drives, 1))
    expect(lambda: c.mseq_wait_device(), "without the flag VO_MSEQ_DEVICE_RESULTS")
    recs = c.mseq_wait()
    for q, w in enumerate(want[0][0]):
        assert all(recs[q][f] == w[f] for f in INTS) and np.array_equal(recs[q]["tvec"], w["tvec"])
    c.close()

def C_byref(r):
    import ctypes
    return ctypes.byref(r)

# ---- launch counts -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mono", [False, True])
def test_launch_counts(built, mono):
    drives = [_drive(640, 240, 31 + q) for q in range(4)]

    def counts(flagged):
        c = _fresh()
        per_sub, per_wait = [], []
        for rep in range(2):                        # the first pass captures the graphs
            per_sub, per_wait = [], []
            c.mseq_begin_device(*_pair(drives, 0), *_mats(drives), mono_rotation=mono, device_results=flagged)
            for k in range(1, NF):
                a = c.kernel_launches()
                c.mseq_submit_device(*_pair(drives, k))
                b = c.kernel_launches()
                if flagged:
                    c.mseq_wait_device()
                else:
                    c.mseq_wait(mono=mono)
                per_sub.append(b - a); per_wait.append(c.kernel_launches() - b)
        torch.cuda.synchronize()
        c.close()
        return per_sub, per_wait
    host_sub, host_wait = counts(False)
    dev_sub, dev_wait = counts(True)
    assert dev_sub == host_sub == [50 if mono else 31] * (NF - 1), (host_sub, dev_sub)
    assert host_wait == [0] * (NF - 1) and dev_wait == [1] * (NF - 1)
