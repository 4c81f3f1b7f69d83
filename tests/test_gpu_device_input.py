"""Images already in GPU memory (vo_seq_*_device, vo_batch_submit_device) through the torch bindings: every record, point
list, pose and carried state is bit-identical to the same pixels through the host entry points -- gray, BGR / RGB
interleaved and planar, pitched and odd-offset slices, the mono_rotation branch, two batch ranges in flight -- and the
stream contract holds: an image produced on the caller's stream right before the call and overwritten right after it
gives the undisturbed results."""
import ctypes as C

import numpy as np
import pytest

from visual_odom_b200 import capi, synth

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

STEP_R = np.array([0.001, -0.004, 0.0005])
STEP_T = np.array([0.01, -0.003, -0.2])
INTS = ("n_features", "n_detected", "n_tracked", "n_valid", "n_inliers", "ransac_iters", "pnp_status")


@pytest.fixture(scope="module")
def dctx(built):
    c = capi.Context(0, max_features=8192)
    yield c
    c.close()


def _frames(w, h, seed, n):
    base = synth.stereo_unit(w, h, seed)
    out = [(base["l0"], base["r0"])]
    for k in range(1, n):
        u = synth.stereo_unit(w, h, seed, rvec=STEP_R * k, tvec=STEP_T * k)
        out.append((u["l1"], u["r1"]))
    return base, out


def _colourise(gray, seed):
    rng = np.random.default_rng(seed)
    tint = rng.integers(-20, 21, gray.shape + (3,))
    return np.clip(gray[..., None].astype(np.int32) + tint, 0, 255).astype(np.uint8)


def _gray_of(bgr):
    b, g, r = (bgr[..., k].astype(np.int64) for k in range(3))
    return ((b * 3735 + g * 19235 + r * 9798 + (1 << 14)) >> 15).astype(np.uint8)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _same(got, ref, what):
    for k in INTS:
        assert got[k] == ref[k], (what, k)
    for k in ("l0", "r0", "l1", "r1", "R", "tvec", "rvec"):
        assert np.array_equal(got[k], ref[k]), (what, k)
    if "mono" in ref:
        for k in ("status", "n_inliers", "ransac_iters", "n_good"):
            assert got["mono"][k] == ref["mono"][k], (what, k)
        assert np.array_equal(got["mono"]["R"], ref["mono"]["R"]) and np.array_equal(got["ess_mask"], ref["ess_mask"]), what


def _host_run(c, base, frames, colour=False, mono=False):
    if colour:
        c.seq_begin_bgr(frames[0][0], frames[0][1], base["P_l"], base["P_r"])
        recs = [c.seq_push_bgr(l, r) for l, r in frames[1:]]
    else:
        c.seq_begin(frames[0][0], frames[0][1], base["P_l"], base["P_r"])
        recs = [c.seq_push(l, r, mono=mono) for l, r in frames[1:]]
    return recs, c.seq_pose(), c.seq_state()


def _check_tail(c, ref):
    recs, pose, state = ref
    assert np.array_equal(c.seq_pose(), pose)
    assert all(np.array_equal(a, b) for a, b in zip(c.seq_state(), state))


@pytest.fixture(scope="module")
def gray_seq(dctx):
    base, frames = _frames(1241, 376, 7, 10)
    return base, frames, _host_run(dctx, base, frames)


def test_gray_push_and_pipelined_submit_equal_host_push(dctx, gray_seq):
    base, frames, ref = gray_seq
    dev = [(_dev(l), _dev(r)) for l, r in frames]
    dctx.seq_begin_device(dev[0][0], dev[0][1], base["P_l"], base["P_r"])
    for k, (l, r) in enumerate(dev[1:]):
        _same(dctx.seq_push_device(l, r), ref[0][k], ("push", k))
    _check_tail(dctx, ref)
    # two frames in flight
    dctx.seq_begin_device(dev[0][0], dev[0][1], base["P_l"], base["P_r"])
    dctx.seq_submit_device(*dev[1])
    for k in range(1, len(dev)):
        if k + 1 < len(dev):
            dctx.seq_submit_device(*dev[k + 1])
            if k == 1:
                with pytest.raises(capi.VoError, match="in flight"):
                    dctx.seq_submit_device(*dev[k + 1])
        _same(dctx.seq_wait(), ref[0][k - 1], ("submit", k))
    _check_tail(dctx, ref)
    assert ref[0][-1]["n_inliers"] > 20


@pytest.mark.parametrize("w,h", [(1241, 376), (637, 241)])
def test_colour_layouts_equal_host_bgr(dctx, w, h):
    base, gray = _frames(w, h, 31, 5)
    bgr = [(_colourise(l, 2 * i), _colourise(r, 2 * i + 1)) for i, (l, r) in enumerate(gray)]
    ref = _host_run(dctx, base, bgr, colour=True)

    def pitched(a):                       # a column slice of a wider tensor: odd base offset, row pitch != 3 w
        big = torch.zeros(a.shape[0], a.shape[1] + 7, 3, dtype=torch.uint8, device="cuda")
        big[:, 3:3 + a.shape[1]] = _dev(a)
        return big[:, 3:3 + a.shape[1]]
    layouts = {
        "bgr_hwc": (lambda a: _dev(a), "bgr"),
        "rgb_hwc": (lambda a: _dev(a[..., ::-1]), "rgb"),
        "rgb_chw": (lambda a: _dev(a[..., ::-1]).permute(2, 0, 1).contiguous(), "rgb"),
        "bgr_pitched": (pitched, "bgr"),
    }
    for name, (make, order) in layouts.items():
        dev = [(make(l), make(r)) for l, r in bgr]
        if name == "bgr_pitched":
            assert dev[0][0].data_ptr() % 2 == 1 and dev[0][0].stride(0) == 3 * (w + 7)
        dctx.seq_begin_device(dev[0][0], dev[0][1], base["P_l"], base["P_r"], order=order)
        for k, (l, r) in enumerate(dev[1:]):
            _same(dctx.seq_push_device(l, r, order=order), ref[0][k], (name, k))
        _check_tail(dctx, ref)


def test_mono_rotation_device_gray_equals_host_gray(built):
    c = capi.Context(0, max_features=8192)
    c.set_option("mono_rotation", 1)
    base, frames = _frames(1241, 376, 23, 5)
    ref = _host_run(c, base, frames, mono=True)
    dev = [(_dev(l), _dev(r)) for l, r in frames]
    c.seq_begin_device(dev[0][0], dev[0][1], base["P_l"], base["P_r"])
    for k, (l, r) in enumerate(dev[1:]):
        _same(c.seq_push_device(l, r, mono=True), ref[0][k], ("mono", k))
    _check_tail(c, ref)
    assert ref[0][-1]["mono"]["status"] == capi.VO_OK
    c.close()


def _batch_units(w, h):
    """Range A (detect): a gray and a BGR unit; range B (given points): a planar RGB and a gray unit.  Returns the host
    units (gray pixels) and the device units with their pixels still as numpy arrays in the device layout."""
    host, dev = [], []
    rng = np.random.default_rng(5)
    for i in range(4):
        u = synth.stereo_unit(w, h, 40 + i, rvec=STEP_R * (i + 1), tvec=STEP_T * (i + 1))
        colour = i in (1, 2)
        imgs = {k: (_colourise(u[k], 10 * i + j) if colour else u[k]) for j, k in enumerate(("l0", "r0", "l1", "r1"))}
        if i < 2:
            extra = dict(n_select=1500)
        else:
            extra = dict(pts=rng.uniform((30, 30), (w - 30, h - 30), (900, 2)).astype(np.float32))
        extra["t_prev"] = tuple(STEP_T)
        host.append(dict({k: (_gray_of(v) if colour else v) for k, v in imgs.items()}, **extra))
        if i == 2:
            d = {k: np.ascontiguousarray(v[..., ::-1].transpose(2, 0, 1)) for k, v in imgs.items()}
            d["order"] = "rgb"
        else:
            d = dict(imgs, order="bgr")
        dev.append(dict(d, **extra))
    return host, dev


def _on_device(units):
    return [dict(u, **{k: _dev(u[k]) for k in ("l0", "r0", "l1", "r1")}) for u in units]


def _batch_results(c, submit, n=4):
    c.set_option("batch_outputs", 1)
    submit(0)
    submit(2)
    recs = np.concatenate([c.batch_wait(0, 2, raw=True), c.batch_wait(2, 2, raw=True)])
    outs = [c.batch_outputs(u, c.records_to_dicts(recs[u:u + 1])[0]) for u in range(n)]
    return recs, outs


def _same_batch(got, ref):
    for f in capi.RESULT_DTYPE.names:
        assert np.array_equal(got[0][f], ref[0][f]), f
    for u, (a, b) in enumerate(zip(got[1], ref[1])):
        for k in ("l0", "r0", "l1", "r1", "kept_idx", "X", "inliers"):
            assert np.array_equal(a[k], b[k]), (u, k)


def test_batch_device_units_equal_host_units(dctx):
    w, h = 1241, 376
    host, dev = _batch_units(w, h)
    base = synth.stereo_unit(w, h, 40)
    dctx.batch_configure(w, h, 4, base["P_l"], base["P_r"])
    keep = []

    def host_submit(u0):
        arr, k, pitch = dctx.make_units(host[u0:u0 + 2])
        keep.append((arr, k))
        dctx.batch_submit(arr, u0, pitch)
    ref = _batch_results(dctx, host_submit)
    dev = _on_device(dev)
    got = _batch_results(dctx, lambda u0: dctx.batch_submit_device(dev[u0:u0 + 2], u0))
    _same_batch(got, ref)
    assert all(r["n_inliers"] > 20 for r in dctx.records_to_dicts(ref[0]))
    assert ref[0]["n_detected"][0] > 0 and ref[0]["n_detected"][2] == 0


def test_stream_ordering_without_host_synchronise(dctx, gray_seq):
    """The image is written on the context's stream right before the call (a non-blocking copy behind a long sleep) and
    zeroed right after it returns; nothing synchronises the host with the stream."""
    base, frames, ref = gray_seq
    s = torch.cuda.Stream()
    pinned = [(torch.from_numpy(l).pin_memory(), torch.from_numpy(r).pin_memory()) for l, r in frames]
    with torch.cuda.stream(s):
        dl = torch.empty(frames[0][0].shape, dtype=torch.uint8, device="cuda")
        dr = torch.empty_like(dl)

        def produce(k):
            torch.cuda._sleep(20_000_000)
            dl.copy_(pinned[k][0], non_blocking=True)
            dr.copy_(pinned[k][1], non_blocking=True)
        produce(0)
        dctx.seq_begin_device(dl, dr, base["P_l"], base["P_r"])
        dl.zero_(); dr.zero_()
        produce(1)
        dctx.seq_submit_device(dl, dr)
        dl.zero_(); dr.zero_()
        for k in range(1, len(frames)):
            if k + 1 < len(frames):
                produce(k + 1)
                dctx.seq_submit_device(dl, dr)
                dl.zero_(); dr.zero_()
            _same(dctx.seq_wait(), ref[0][k - 1], ("stream", k))
        _check_tail(dctx, ref)

        # the batched mode, two ranges in flight
        w, h = 1241, 376
        host, dev = _batch_units(w, h)
        dctx.batch_configure(w, h, 4, base["P_l"], base["P_r"])
        keep = []

        def host_submit(u0):
            arr, kp, pitch = dctx.make_units(host[u0:u0 + 2])
            keep.append((arr, kp))
            dctx.batch_submit(arr, u0, pitch)
        want = _batch_results(dctx, host_submit)
        src = [{k: torch.from_numpy(d[k]).pin_memory() for k in ("l0", "r0", "l1", "r1")} for d in dev]
        bufs = [{k: torch.empty(d[k].shape, dtype=torch.uint8, device="cuda") for k in ("l0", "r0", "l1", "r1")} for d in src]

        def dev_submit(u0):
            torch.cuda._sleep(20_000_000)
            for u in (u0, u0 + 1):
                for k in ("l0", "r0", "l1", "r1"):
                    bufs[u][k].copy_(src[u][k], non_blocking=True)
            dctx.batch_submit_device([dict(dev[u], **bufs[u]) for u in (u0, u0 + 1)], u0)
            for u in (u0, u0 + 1):
                for t in bufs[u].values():
                    t.zero_()
        _same_batch(_batch_results(dctx, dev_submit), want)


def test_refusals_leave_the_context_usable(dctx, gray_seq):
    base, frames, ref = gray_seq
    lib = dctx.lib
    w, h = 1241, 376
    dl, dr = _dev(frames[0][0]), _dev(frames[0][1])
    good, _, _ = capi.image_descriptor(dl.shape, dl.stride(), dl.data_ptr())
    host = np.ascontiguousarray(frames[1][0])
    pinned = torch.from_numpy(host).pin_memory()
    P_l = np.ascontiguousarray(base["P_l"], np.float32).reshape(12); P_r = np.ascontiguousarray(base["P_r"], np.float32).reshape(12)

    def bad(**kw):
        d = capi.VoDImage.from_buffer_copy(good)
        for k, v in kw.items():
            setattr(d, k, v)
        return d
    dctx.batch_configure(w, h, 2, base["P_l"], base["P_r"])
    units = (capi.VoDUnit * 1)()
    for k in ("l0", "r0", "l1", "r1"):
        setattr(units[0], k, good)
    units[0].r1 = bad(data=pinned.data_ptr())
    units[0].n_pts = 100
    assert lib.vo_batch_submit_device(dctx.h, units, 0, 1) == capi.VO_E_INVALID
    assert "pinned host" in lib.vo_last_error(dctx.h).decode()
    dctx.seq_begin_device(dl, dr, base["P_l"], base["P_r"])
    cases = [(bad(data=host.ctypes.data), "host"), (bad(data=pinned.data_ptr()), "pinned host"),
             (bad(row_pitch=w - 1), "row_pitch"), (bad(format=7), "unknown format"), (bad(pixel_stride=0), "pixel_stride")]
    for d, msg in cases:
        rc = lib.vo_seq_submit_device(dctx.h, C.byref(good), C.byref(d))
        assert rc == capi.VO_E_INVALID and msg in lib.vo_last_error(dctx.h).decode(), msg
        rc = lib.vo_seq_begin_device(dctx.h, w, h, capi._p(P_l), capi._p(P_r), C.byref(d), C.byref(good))
        assert rc == capi.VO_E_INVALID and msg in lib.vo_last_error(dctx.h).decode(), msg
    # the refused calls changed nothing: the same sequence gives the reference results
    dev = [(_dev(l), _dev(r)) for l, r in frames]
    dctx.seq_begin_device(dev[0][0], dev[0][1], base["P_l"], base["P_r"])
    for k, (l, r) in enumerate(dev[1:]):
        _same(dctx.seq_push_device(l, r), ref[0][k], ("after refusals", k))
    _check_tail(dctx, ref)
