"""Multi-sequence runs fed from images already in GPU memory (vo_mseq_begin_device / vo_mseq_submit_device) through the
torch bindings: every sequence is, frame by frame, bit-identical to the same pixels through the host vo_mseq_* entry
points -- records, the four point lists, the carried FeatureSet and translation, frame_pose, and with
VO_MSEQ_MONO_ROTATION the mono results and essential masks.  The cases: gray drives of two sizes (submit-then-wait and
two in flight), mixed layouts in one submission (gray, BGR / RGB interleaved, RGB planar, an odd-offset column slice, the
two bytes of a 16-bit stereo buffer), KITTI's three sizes and cameras, the mono branch, retirement and starts into empty,
retired and live slots (a smaller start into a larger slot with another submission in flight), host and device
submissions alternating, the stream contract, graphs off, launch counts, and every refusal."""

import numpy as np
import pytest

from visual_odom_b200 import capi, synth

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
cv2 = pytest.importorskip("cv2")

K0 = synth.KITTI00
INTS = ("n_features", "n_detected", "n_tracked", "n_valid", "n_inliers", "ransac_iters", "pnp_status", "status")
ARRAYS = ("rvec", "tvec", "R", "l0", "r0", "l1", "r1")
NF = 4                      # frames per drive: the first pair and three submissions

def _cal(sx=1.0, dcx=0.0, dcy=0.0, sb=1.0):
    return dict(fx=K0["fx"] * sx, fy=K0["fy"] * sx, cx=K0["cx"] + dcx, cy=K0["cy"] + dcy, bf=K0["bf"] * sb)

_FRAMES = {}

def _drive(w, h, seed, cal=None, n=NF, step_r=(0.001, -0.004, 0.0005), step_t=(0.01, -0.003, -0.2)):
    """(P_l, P_r, [(left, right)] * n): gray frames of one synthetic drive."""
    cal = cal or _cal(1.0, (w - 1241) / 2.0, (h - 376) / 2.0)
    key = (w, h, seed, tuple(sorted(cal.items())), n, step_r, step_t)
    if key not in _FRAMES:
        base = synth.stereo_unit(w, h, seed, cal=cal)
        fr = [(base["l0"], base["r0"])]
        for k in range(1, n):
            u = synth.stereo_unit(w, h, seed, cal=cal, rvec=np.array(step_r) * k, tvec=np.array(step_t) * k)
            fr.append((u["l1"], u["r1"]))
        _FRAMES[key] = (base["P_l"], base["P_r"], fr)
    return _FRAMES[key]

def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()

@pytest.fixture(scope="module")
def mctx(built):
    c = capi.Context(0, max_features=8192)
    yield c
    c.close()

def _collect(ctx, n, mono, full):
    recs = ctx.mseq_wait(mono=mono)
    if not full:
        return recs, None, None
    return recs, [ctx.mseq_state(q) for q in range(n)], [ctx.mseq_pose(q) for q in range(n)]

def _run(ctx, n, begin, submits, mono=False, pipelined=False):
    """begin(); then submits[k]() for every submission k, waited one by one (with every sequence's state and pose after
    each wait) or two in flight (records only)."""
    begin()
    out = []
    if pipelined:
        submits[0]()
        for k in range(len(submits)):
            if k + 1 < len(submits):
                submits[k + 1]()
            out.append(_collect(ctx, n, mono, False))
        return out
    for s in submits:
        s()
        out.append(_collect(ctx, n, mono, True))
    return out

def _same_runs(got, want, what=""):
    assert len(got) == len(want)
    for k, ((ga, gs, gp), (wa, ws, wp)) in enumerate(zip(got, want)):
        for q, (a, b) in enumerate(zip(ga, wa)):
            where = f"{what} submission {k} sequence {q}"
            for f in INTS:
                assert a[f] == b[f], f"{where}: {f} {a[f]} != {b[f]}"
            for f in ARRAYS:
                assert a[f].dtype == b[f].dtype and np.array_equal(a[f], b[f]), f"{where}: {f}"
            if "mono" in b:
                for f in ("status", "n_inliers", "ransac_iters", "n_good"):
                    assert a["mono"][f] == b["mono"][f], f"{where}: mono {f}"
                assert np.array_equal(a["mono"]["R"], b["mono"]["R"]) and np.array_equal(a["ess_mask"], b["ess_mask"]), where
        if ws is not None:
            for q, (x, y) in enumerate(zip(gs, ws)):
                assert all(np.array_equal(u, v) for u, v in zip(x, y)), f"{what} submission {k}: state of sequence {q}"
            for q, (x, y) in enumerate(zip(gp, wp)):
                assert np.array_equal(x, y), f"{what} submission {k}: pose of sequence {q}"

def _host_lockstep(ctx, drives, mono=False, pipelined=False, gray=None):
    """The drives (lists of (P_l, P_r, frames)) through mseq_begin / mseq_submit; gray(q, img) = the host gray pixels of
    sequence q's image (default: the frames themselves)."""
    n = len(drives)
    gray = gray or (lambda q, a: a)
    P_l = np.stack([d[0] for d in drives]); P_r = np.stack([d[1] for d in drives])

    def pair(k):
        return [gray(q, d[2][k][0]) for q, d in enumerate(drives)], [gray(q, d[2][k][1]) for q, d in enumerate(drives)]
    return _run(ctx, n, lambda: ctx.mseq_begin(*pair(0), P_l, P_r, mono_rotation=mono),
                [lambda k=k: ctx.mseq_submit(*pair(k)) for k in range(1, NF)], mono, pipelined)

def _device_lockstep(ctx, drives, mono=False, pipelined=False, layout=None, order=None):
    """The same through mseq_begin_device / mseq_submit_device; layout(q, img) = sequence q's CUDA tensor of a frame."""
    n = len(drives)
    layout = layout or (lambda q, a: _dev(a))
    P_l = np.stack([d[0] for d in drives]); P_r = np.stack([d[1] for d in drives])
    dev = [[(layout(q, l), layout(q, r)) for l, r in d[2]] for q, d in enumerate(drives)]

    def pair(k):
        return [dev[q][k][0] for q in range(n)], [dev[q][k][1] for q in range(n)]
    return _run(ctx, n, lambda: ctx.mseq_begin_device(*pair(0), P_l, P_r, order=order, mono_rotation=mono),
                [lambda k=k: ctx.mseq_submit_device(*pair(k), order=order) for k in range(1, NF)], mono, pipelined)

GRAY_DRIVES = [(640, 240, 31), (640, 240, 7), (640, 240, 13), (640, 240, 42), (640, 240, 5), (1241, 376, 11), (1241, 376, 23)]

def test_gray_drives_equal_the_host_path(mctx):
    drives = [_drive(w, h, s) for w, h, s in GRAY_DRIVES]
    for pipelined in (False, True):
        want = _host_lockstep(mctx, drives, pipelined=pipelined)
        _same_runs(_device_lockstep(mctx, drives, pipelined=pipelined), want, f"pipelined={pipelined}")
    assert all(r["n_inliers"] > 20 for r in want[-1][0])

def _cvt(a, code):
    return cv2.cvtColor(np.ascontiguousarray(a), code)

def _colourise(gray, seed):
    rng = np.random.default_rng(seed)
    tint = rng.integers(-20, 21, gray.shape + (3,))
    return np.clip(gray[..., None].astype(np.int32) + tint, 0, 255).astype(np.uint8)

def test_mixed_layouts_in_one_submission_equal_the_host_gray_of_their_pixels(mctx):
    """Sequence q's frames are colour images (BGR pixels b) in q's own layout; the host reference is the gray run of
    cv2.cvtColor(b, BGR2GRAY).  The last sequence is one 640 x 480 16-bit buffer per frame whose low bytes are the left
    image and whose high bytes are the right image, passed as two gray images at data / data + 1 with pixel stride 2."""
    drives = [_drive(640, 240, s) for s in (31, 7, 13, 42, 5)] + [_drive(640, 480, 17)]
    colour = {}

    def bgr(q, a):
        k = id(a)
        if k not in colour:
            colour[k] = _colourise(a, len(colour) + 97 * q)
        return colour[k]

    def pitched(b):
        big = torch.zeros(b.shape[0], b.shape[1] + 7, 3, dtype=torch.uint8, device="cuda")
        big[:, 3:3 + b.shape[1]] = _dev(b)
        return big[:, 3:3 + b.shape[1]]                  # base offset 9 bytes, row pitch 3 (w + 7)
    layouts = [lambda b: _dev(_cvt(b, cv2.COLOR_BGR2GRAY)),                        # gray
               lambda b: _dev(b),                                                   # BGR HWC
               lambda b: _dev(b[..., ::-1]),                                        # RGB HWC
               lambda b: _dev(b[..., ::-1]).permute(2, 0, 1).contiguous(),         # RGB CHW
               pitched]                                                             # BGR HWC column slice, odd offset
    orders = ["bgr", "bgr", "rgb", "rgb", "bgr", None]

    def dev_pairs(q, d):
        if q < 5:
            return [(layouts[q](bgr(q, l)), layouts[q](bgr(q, r))) for l, r in d[2]]
        out = []
        for l, r in d[2]:
            buf = torch.from_numpy((l.astype(np.uint16) | (r.astype(np.uint16) << 8)).view(np.int16)).cuda()
            v = buf.view(torch.uint8)                      # (480, 1280): little-endian, the left byte first
            out.append((v[:, 0::2], v[:, 1::2]))
        return out

    n = len(drives)
    P_l = np.stack([d[0] for d in drives]); P_r = np.stack([d[1] for d in drives])
    dev = [dev_pairs(q, d) for q, d in enumerate(drives)]
    assert dev[5][0][1].data_ptr() == dev[5][0][0].data_ptr() + 1 and dev[5][0][0].stride() == (1280, 2)

    def pair(k):
        return [dev[q][k][0] for q in range(n)], [dev[q][k][1] for q in range(n)]
    got = _run(mctx, n, lambda: mctx.mseq_begin_device(*pair(0), P_l, P_r, order=orders),
               [lambda k=k: mctx.mseq_submit_device(*pair(k), order=orders) for k in range(1, NF)])
    want = _host_lockstep(mctx, drives, gray=lambda q, a: _cvt(bgr(q, a), cv2.COLOR_BGR2GRAY) if q < 5 else a)
    _same_runs(got, want, "layouts")
    assert all(r["n_inliers"] > 20 for r in want[-1][0])

def test_kitti_sizes_and_cameras_equal_the_host_sized_run(mctx):
    drives = [_drive(1241, 376, 3, _cal()), _drive(1242, 375, 4, _cal(0.98, 0.5, -0.5, 1.02)),
              _drive(1226, 370, 6, _cal(1.01, -7.5, -3.0, 0.97))]
    for pipelined in (False, True):
        _same_runs(_device_lockstep(mctx, drives, pipelined=pipelined), _host_lockstep(mctx, drives, pipelined=pipelined),
                   f"kitti pipelined={pipelined}")

def test_mono_rotation_equals_the_host_run(mctx):
    drives = [_drive(640, 240, s) for s in (31, 7)] + [_drive(601, 233, 13)]
    want = _host_lockstep(mctx, drives, mono=True)
    _same_runs(_device_lockstep(mctx, drives, mono=True), want, "mono")
    assert all(r["mono"]["status"] == 0 for r in want[-1][0])

# ---- slots: retirement, starts, alternation -------------------------------------------------------------------------
ENV = (656, 248)
# (slot, first submission, drive, frames): slot 0 runs a 656 x 248 drive, is retired by a NULL pair at submission 4 and
# gets a smaller 512 x 200 drive at 5 (two in flight: its geometry changes under the frame in flight); slot 1's live drive
# is replaced at 3 by a drive with another camera; slot 2 starts empty at 2; slot 3 stays empty throughout.
SLOT_DRIVES = {"a": (656, 248, 13), "b": (512, 200, 42), "c": (640, 240, 31), "d": (601, 233, 7), "e": (620, 236, 23)}
SCHED = [(0, 1, "a", 3), (0, 5, "b", 3), (1, 1, "c", 2), (1, 3, "d", 4), (2, 2, "e", 5)]
N_SLOTS, K_LAST = 4, 7

def _slot_run(ctx, use_device, pipelined=False, mono=False):
    """The schedule through mseq_open; use_device(k) picks device tensors for submission k."""
    frames = {k: _drive(*v, n=5) for k, v in SLOT_DRIVES.items()}
    dev = {k: [(_dev(l), _dev(r)) for l, r in v[2]] for k, v in frames.items()}

    def go(k):
        dv = use_device(k)
        lefts, rights, start = [None] * N_SLOTS, [None] * N_SLOTS, {}
        for q, k0, d, L in SCHED:
            if k0 <= k < k0 + L:
                lefts[q], rights[q] = (dev if dv else {d: frames[d][2]})[d][k - k0]
                if k == k0:
                    start[q] = frames[d][:2]
        if dv:
            ctx.mseq_submit_device(lefts, rights, start=start)
        else:
            ctx.mseq_submit(lefts, rights, start=start)
    return _run(ctx, N_SLOTS, lambda: ctx.mseq_open(N_SLOTS, *ENV, mono_rotation=mono),
                [lambda k=k: go(k) for k in range(1, K_LAST + 1)], mono, pipelined)

@pytest.mark.parametrize("pipelined", [False, True])
def test_retirement_and_starts_equal_host_starts(mctx, pipelined):
    want = _slot_run(mctx, lambda k: False, pipelined)
    _same_runs(_slot_run(mctx, lambda k: True, pipelined), want, "device starts")
    st = [[r["status"] for r in recs] for recs, _, _ in want]
    assert st[0] == [capi.VO_MSEQ_STARTED, capi.VO_MSEQ_STARTED, capi.VO_MSEQ_RETIRED, capi.VO_MSEQ_RETIRED]
    assert st[3][0] == capi.VO_MSEQ_RETIRED and st[4][0] == capi.VO_MSEQ_STARTED and st[2][1] == capi.VO_MSEQ_STARTED
    assert all(recs[3]["status"] == capi.VO_MSEQ_RETIRED for recs, _, _ in want)
    assert max(r["n_inliers"] for recs, _, _ in want for r in recs) > 20

@pytest.mark.parametrize("pipelined", [False, True])
def test_host_and_device_submissions_alternate(mctx, pipelined):
    want = _slot_run(mctx, lambda k: False, pipelined)
    _same_runs(_slot_run(mctx, lambda k: k % 2 == 0, pipelined), want, "even device")
    _same_runs(_slot_run(mctx, lambda k: k % 2 == 1, pipelined), want, "odd device")

def test_graphs_off_equals_graphs_on(mctx):
    drives = [_drive(640, 240, 31), _drive(601, 233, 7)]
    want = _device_lockstep(mctx, drives, pipelined=True)
    mctx.set_option("graphs", 0)
    try:
        got = _device_lockstep(mctx, drives, pipelined=True)
        slots = _slot_run(mctx, lambda k: True, True)
    finally:
        mctx.set_option("graphs", 1)
    _same_runs(got, want, "graphs=0")
    _same_runs(slots, _slot_run(mctx, lambda k: True, True), "slots graphs=0")

# ---- stream contract -----------------------------------------------------------------------------------------------
def test_images_produced_right_before_and_overwritten_right_after_the_call(mctx):
    """Every source tensor is written by a kernel on the current stream just before the call and overwritten with noise
    on the same stream just after it, with no host synchronise: the results are those of the undisturbed pixels."""
    drives = [_drive(640, 240, 31), _drive(601, 233, 7), _drive(640, 240, 13)]
    want = _host_lockstep(mctx, drives, pipelined=True)
    n = len(drives)
    key = torch.tensor(0x5A, dtype=torch.uint8, device="cuda")
    # the frames xor-ed with a key, and one scratch tensor per image of a submission (two submissions in flight)
    enc = [[(_dev(l) ^ key, _dev(r) ^ key) for l, r in d[2]] for d in drives]
    scratch = [[(torch.empty_like(enc[q][0][0]), torch.empty_like(enc[q][0][1])) for q in range(n)] for _ in range(2)]
    g = torch.Generator(device="cuda")
    g.manual_seed(5)

    def produced(k):
        buf = scratch[k % 2]
        for q in range(n):
            for i in range(2):
                torch.bitwise_xor(enc[q][k][i], key, out=buf[q][i])
        return [b[0] for b in buf], [b[1] for b in buf]

    def clobber(k):
        for b in scratch[k % 2]:
            for t in b:
                t.random_(generator=g)

    def begin():
        mctx.mseq_begin_device(*produced(0), np.stack([d[0] for d in drives]), np.stack([d[1] for d in drives]))
        clobber(0)

    def submit(k):
        mctx.mseq_submit_device(*produced(k))
        clobber(k)
    _same_runs(_run(mctx, n, begin, [lambda k=k: submit(k) for k in range(1, NF)], pipelined=True), want, "stream contract")

# ---- launch counts -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_seq", [1, 16])
def test_a_device_submission_costs_one_launch_more_than_a_host_gray_one(mctx, n_seq):
    drives = [_drive(640, 240, 31 + q) for q in range(n_seq)]

    def per_submission(device):
        cnt = []
        P_l = np.stack([d[0] for d in drives]); P_r = np.stack([d[1] for d in drives])
        if device:
            dev = [[(_dev(l), _dev(r)) for l, r in d[2]] for d in drives]
            mctx.mseq_begin_device([d[0][0] for d in dev], [d[0][1] for d in dev], P_l, P_r)
        else:
            mctx.mseq_begin([d[2][0][0] for d in drives], [d[2][0][1] for d in drives], P_l, P_r)
        for k in range(1, NF):
            before = mctx.kernel_launches()
            if device:
                mctx.mseq_submit_device([d[k][0] for d in dev], [d[k][1] for d in dev])
            else:
                mctx.mseq_submit([d[2][k][0] for d in drives], [d[2][k][1] for d in drives])
            mctx.mseq_wait()
            cnt.append(mctx.kernel_launches() - before)
        return cnt
    per_submission(False); per_submission(True)         # graphs captured
    host, dev = per_submission(False), per_submission(True)
    assert dev == [c + 1 for c in host], (host, dev)

# ---- refusals ------------------------------------------------------------------------------------------------------
def _raw_submit(ctx, lefts, rights, starts=()):
    """vo_mseq_submit_device with hand-made descriptors (through the binding's stream handling)."""
    n = len(lefts)
    lt, rt = (capi.VoDImage * n)(*lefts), (capi.VoDImage * n)(*rights)
    arr, ns = ctx._starts(dict(starts)) if starts else (None, 0)
    ctx._device_call(ctx.lib.vo_mseq_submit_device, lt, rt, ns, arr)

def _gray_desc(t):
    return capi.image_descriptor(t.shape, t.stride(), t.data_ptr())[0]

def test_refusals_change_nothing(built, mctx):
    drives = [_drive(640, 240, 31), _drive(601, 233, 7), _drive(640, 240, 13)]
    n = len(drives)
    P_l = np.stack([d[0] for d in drives]); P_r = np.stack([d[1] for d in drives])
    want = _host_lockstep(mctx, drives, pipelined=True)
    dev = [[(_dev(l), _dev(r)) for l, r in d[2]] for d in drives]

    def pair(k):
        return [dev[q][k][0] for q in range(n)], [dev[q][k][1] for q in range(n)]

    def descs(k):
        return [_gray_desc(t) for t in pair(k)[0]], [_gray_desc(t) for t in pair(k)[1]]
    host = np.ascontiguousarray(drives[0][2][1][0])
    pinned = torch.from_numpy(host).pin_memory()
    other = capi.Context(0, max_features=8192)

    def refusals(k):
        """Every refusal at submission k (one submission in flight), each checked for its code."""
        def expect(code, fn, match=None):
            with pytest.raises(capi.VoError, match=match) as e:
                fn()
            assert e.value.code == code, (e.value.code, str(e.value))

        def with_left(q, d):
            l, r = descs(k)
            l[q] = d
            return l, r
        hd = _gray_desc(pinned); hd.data = host.ctypes.data
        expect(capi.VO_E_INVALID, lambda: _raw_submit(mctx, *with_left(1, hd)), "host")
        expect(capi.VO_E_INVALID, lambda: _raw_submit(mctx, *with_left(0, _gray_desc(pinned))), "pinned host")
        short = _gray_desc(pair(k)[0][1]); short.row_pitch = 600                          # sequence 1 is 601 wide
        expect(capi.VO_E_INVALID, lambda: _raw_submit(mctx, *with_left(1, short)), "row_pitch 600 < 601")
        bad = _gray_desc(pair(k)[0][2]); bad.format = 7
        expect(capi.VO_E_INVALID, lambda: _raw_submit(mctx, *with_left(2, bad)), "unknown format")
        expect(capi.VO_E_INVALID, lambda: _raw_submit(mctx, *with_left(2, capi.VoDImage())), "only one image")
        expect(capi.VO_E_INVALID, lambda: _raw_submit(mctx, *descs(k), starts={3: (640, 240, P_l[0], P_r[0])}), "slot 3")
        expect(capi.VO_E_UNSUPPORTED, lambda: _raw_submit(mctx, *descs(k), starts={0: (640, 250, P_l[0], P_r[0])}), "envelope")
        expect(capi.VO_E_INVALID, lambda: mctx._device_call(mctx.lib.vo_mseq_submit_device, None, None, 0, None), "bad argument")
        expect(capi.VO_E_INVALID, lambda: mctx.seq_submit_device(*[t[0] for t in pair(k)]), "vo_mseq_begin")

    got = _run(mctx, n, lambda: mctx.mseq_begin_device(*pair(0), P_l, P_r), [
        lambda: mctx.mseq_submit_device(*pair(1)),
        lambda: (refusals(2), mctx.mseq_submit_device(*pair(2))),
        lambda: mctx.mseq_submit_device(*pair(3))], pipelined=True)
    _same_runs(got, want, "after refusals")
    # a third submission in flight, a retired sequence's pair, and the other sequence mode's calls
    mctx.mseq_begin_device(*pair(0), P_l, P_r)
    mctx.mseq_submit_device(*pair(1))
    mctx.mseq_submit_device(*pair(2))
    with pytest.raises(capi.VoError, match="in flight") as e:
        mctx.mseq_submit_device(*pair(3))
    assert e.value.code == capi.VO_E_INVALID
    r1, r2 = mctx.mseq_wait(), mctx.mseq_wait()
    _same_runs([(r1, None, None), (r2, None, None)], want[:2], "third in flight")
    l, r = pair(3)
    mctx.mseq_submit_device(l[:2] + [None], r[:2] + [None])
    assert mctx.mseq_wait()[2]["status"] == capi.VO_MSEQ_RETIRED
    with pytest.raises(capi.VoError, match="retired") as e:
        mctx.mseq_submit_device(*pair(3))
    assert e.value.code == capi.VO_E_INVALID
    # vo_mseq_submit_device while vo_seq_* runs, and a begin while a batch submission is pending
    base = drives[0]
    other.seq_begin_device(dev[0][0][0], dev[0][0][1], base[0], base[1])
    with pytest.raises(capi.VoError, match="vo_seq_begin") as e:
        _raw_submit(other, [_gray_desc(dev[0][1][0])], [_gray_desc(dev[0][1][1])])
    assert e.value.code == capi.VO_E_INVALID
    u = synth.stereo_unit(640, 240, 31)
    other.batch_configure(640, 240, 1, u["P_l"], u["P_r"])
    arr, keep, pitch = other.make_units([dict(u, n_select=300, t_prev=(0.0, 0.0, -0.2))])
    other.batch_submit(arr, 0, pitch)
    with pytest.raises(capi.VoError, match="has not been waited for") as e:
        other.mseq_begin_device(*pair(0), P_l, P_r)
    assert e.value.code == capi.VO_E_INVALID
    other.batch_wait(0, 1)
    del keep
    _same_runs(_device_lockstep(other, drives, pipelined=True), want, "after the batch")
    other.close()
