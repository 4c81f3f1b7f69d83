"""ctypes binding of libvo_b200.so (include/vo_b200.h).

This is plumbing only: it loads the in-tree shared library and exposes each C-ABI entry point
with numpy buffers.  There is no Python/CPU implementation behind it -- if the library is
missing or no H100 (compute capability 9.0) is present, the calls fail loudly.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libvo_b200.so")

VO_OK = 0
VO_E_INVALID = -1
VO_E_CUDA = -2
VO_E_TOO_FEW_POINTS = -3
VO_E_UNSUPPORTED = -4
VO_DIST_DEPTH = 8          # gathers that may be outstanding (include/vo_b200.h)
VO_E_CAPACITY = -5
VO_MSEQ_MAX = 64           # sequences one vo_mseq_begin may start (include/vo_b200.h)
VO_MSEQ_RETIRED = 2        # vo_mseq_wait status of a retired sequence
VO_MSEQ_MONO_ROTATION = 1  # vo_mseq_begin_ex flag: every sequence runs trackingFrame2Frame(mono_rotation = true)
VO_MSEQ_STARTED = 3        # vo_mseq_wait status of the submission that started a slot's sequence
VO_MSEQ_DEVICE_RESULTS = 8 # vo_mseq_begin* / vo_mseq_open flag: results into device memory through vo_mseq_wait_device


class VoParams(C.Structure):
    _fields_ = [
        ("fast_threshold", C.c_int), ("fast_nonmax", C.c_int), ("lk_win", C.c_int),
        ("lk_max_level", C.c_int), ("lk_max_iters", C.c_int), ("lk_epsilon", C.c_double),
        ("lk_min_eig", C.c_double), ("circ_threshold", C.c_int), ("pnp_iterations", C.c_int),
        ("pnp_reproj_error", C.c_float), ("pnp_confidence", C.c_double),
        ("max_features", C.c_int), ("max_units", C.c_int),
        # the sequence modes' bookkeeping (matchingFeatures' literals); the batched path ignores them
        ("refill_threshold", C.c_int), ("bucket_rows_divisor", C.c_int), ("features_per_bucket", C.c_int),
        ("bucket_age_threshold", C.c_int),
    ]


class VoUnit(C.Structure):
    _fields_ = [
        ("l0", C.c_void_p), ("r0", C.c_void_p), ("l1", C.c_void_p), ("r1", C.c_void_p),
        ("pts", C.c_void_p), ("n_pts", C.c_int), ("t_prev", C.c_double * 3),
    ]


VO_FMT_GRAY, VO_FMT_BGR, VO_FMT_RGB = 0, 1, 2


class VoDImage(C.Structure):
    _fields_ = [("data", C.c_void_p), ("row_pitch", C.c_size_t), ("pixel_stride", C.c_int), ("channel_stride", C.c_size_t),
                ("format", C.c_int)]


class VoDUnit(C.Structure):
    _fields_ = [("l0", VoDImage), ("r0", VoDImage), ("l1", VoDImage), ("r1", VoDImage),
                ("pts", C.c_void_p), ("n_pts", C.c_int), ("t_prev", C.c_double * 3)]


def image_descriptor(shape, strides, data_ptr, order=None):
    """The vo_dimage of a uint8 image laid out (H, W), (H, W, 3) or (3, H, W) with the given byte strides (as torch's
    t.shape, t.stride() and t.data_ptr() of a uint8 tensor give them).  Returns (VoDImage, w, h).  Colour images need
    order="bgr" or "rgb"; there is no default.  Raises ValueError for any other layout, for non-positive strides and for
    rows that overlap (a transposed image)."""
    shape, strides = tuple(int(v) for v in shape), tuple(int(v) for v in strides)
    if len(shape) == 2:
        (h, w), (rs, ps), cs, fmt = shape, strides, 0, VO_FMT_GRAY
    elif len(shape) == 3:
        hwc, chw = shape[2] == 3, shape[0] == 3
        if hwc == chw:
            raise ValueError(f"image of shape {shape}: expected (H, W, 3) or (3, H, W)")
        (h, w), (rs, ps), cs = (shape[:2], strides[:2], strides[2]) if hwc else (shape[1:], strides[1:], strides[0])
        if order not in ("bgr", "rgb"):
            raise ValueError(f'colour image: order must be "bgr" or "rgb" (got {order!r})')
        fmt = VO_FMT_BGR if order == "bgr" else VO_FMT_RGB
        if cs <= 0:
            raise ValueError(f"image strides {strides}: strides must be positive")
    else:
        raise ValueError(f"image of shape {shape}: expected (H, W), (H, W, 3) or (3, H, W)")
    if h <= 0 or w <= 0:
        raise ValueError(f"empty image of shape {shape}")
    if rs <= 0 or ps <= 0:
        raise ValueError(f"image strides {strides}: strides must be positive")
    if rs < w * ps:
        raise ValueError(f"image strides {strides}: rows of {w} pixels overlap (row pitch {rs} < {w} x {ps})")
    d = VoDImage()
    d.data, d.row_pitch, d.pixel_stride, d.channel_stride, d.format = data_ptr, rs, ps, cs, fmt
    return d, w, h


class VoUnitResult(C.Structure):
    _fields_ = [
        ("n_features", C.c_int), ("n_detected", C.c_int), ("n_tracked", C.c_int), ("n_valid", C.c_int),
        ("n_inliers", C.c_int), ("ransac_iters", C.c_int), ("pnp_status", C.c_int),
        ("rvec", C.c_double * 3), ("tvec", C.c_double * 3), ("R", C.c_double * 9),
    ]


class VoMseqStart(C.Structure):
    """vo_mseq_start: the slot, image size and matrices of a sequence that vo_mseq_submit_start starts."""
    _fields_ = [("slot", C.c_int), ("w", C.c_int), ("h", C.c_int), ("P_l", C.c_float * 12), ("P_r", C.c_float * 12)]


class VoMonoResult(C.Structure):
    _fields_ = [
        ("status", C.c_int), ("n_inliers", C.c_int), ("ransac_iters", C.c_int), ("n_good", C.c_int),
        ("R", C.c_double * 9), ("t", C.c_double * 3),
    ]


class VoMseqDResults(C.Structure):
    """vo_mseq_dresults: the caller's device buffers vo_mseq_wait_device writes (any pointer may be NULL)."""
    _fields_ = [("status", C.c_void_p), ("records", C.c_void_p), ("frame_pose", C.c_void_p), ("pts_cap", C.c_int),
                ("pts4", C.c_void_p), ("points3d", C.c_void_p), ("inliers", C.c_void_p), ("mono", C.c_void_p),
                ("ess_mask", C.c_void_p)]


# the same record as a numpy structured dtype (C layout, 152 bytes): arrays of records can be handed out without building
# one Python dict per record (a gathered table of a multi-GPU step has world x units of them)
RESULT_DTYPE = np.dtype([("n_features", "<i4"), ("n_detected", "<i4"), ("n_tracked", "<i4"), ("n_valid", "<i4"), ("n_inliers", "<i4"),
                         ("ransac_iters", "<i4"), ("pnp_status", "<i4"), ("rvec", "<f8", (3,)), ("tvec", "<f8", (3,)),
                         ("R", "<f8", (3, 3))], align=True)
assert RESULT_DTYPE.itemsize == C.sizeof(VoUnitResult)


# name -> (restype, argtypes); every symbol include/vo_b200.h declares must be listed here
SIGNATURES = {
    "vo_default_params": (None, [C.POINTER(VoParams)]),
    "vo_create": (C.c_int, [C.c_int, C.POINTER(VoParams), C.POINTER(C.c_void_p)]),
    "vo_destroy": (None, [C.c_void_p]),
    "vo_last_error": (C.c_char_p, [C.c_void_p]),
    "vo_set_stream": (C.c_int, [C.c_void_p, C.c_void_p]),
    "vo_sync": (C.c_int, [C.c_void_p]),
    "vo_kernel_launches": (C.c_longlong, [C.c_void_p]),
    "vo_lk_kernel_time": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_longlong), C.c_int]),
    "vo_set_option": (C.c_int, [C.c_void_p, C.c_char_p, C.c_double]),
    "vo_fast_detect": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_size_t, C.c_void_p, C.c_void_p,
                                 C.c_int, C.POINTER(C.c_int)]),
    "vo_lk_track": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_size_t, C.c_void_p, C.c_int,
                              C.c_void_p, C.c_void_p, C.c_void_p]),
    "vo_circular_match": (C.c_int, [C.c_void_p] + [C.c_void_p] * 4 + [C.c_int, C.c_int, C.c_size_t, C.c_void_p, C.c_int,
                                    C.c_void_p] + [C.c_void_p] * 5 + [C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.POINTER(C.c_int)]),
    "vo_triangulate": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "vo_triangulate_homogeneous": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "vo_pnp_ransac": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                C.c_void_p, C.POINTER(C.c_int), C.c_void_p, C.POINTER(C.c_int)]),
    "vo_batch_configure": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vo_batch_upload": (C.c_int, [C.c_void_p, C.POINTER(VoUnit), C.c_int, C.c_size_t]),
    "vo_batch_run": (C.c_int, [C.c_void_p]),
    "vo_batch_download": (C.c_int, [C.c_void_p, C.POINTER(VoUnitResult), C.c_int]),
    "vo_frame_batch": (C.c_int, [C.c_void_p, C.POINTER(VoUnit), C.c_int, C.c_size_t, C.POINTER(VoUnitResult)]),
    "vo_batch_submit": (C.c_int, [C.c_void_p, C.POINTER(VoUnit), C.c_int, C.c_int, C.c_size_t]),
    "vo_batch_wait": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(VoUnitResult)]),
    "vo_seq_begin": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "vo_seq_push": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(VoUnitResult), C.c_void_p, C.c_int]),
    "vo_seq_submit": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]),
    "vo_seq_wait": (C.c_int, [C.c_void_p, C.POINTER(VoUnitResult), C.c_void_p, C.c_int]),
    "vo_seq_wait_mono": (C.c_int, [C.c_void_p, C.POINTER(VoUnitResult), C.POINTER(VoMonoResult), C.c_void_p, C.c_int,
                                   C.c_void_p, C.c_int]),
    "vo_seq_state": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_void_p]),
    "vo_seq_begin_ex": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]),
    "vo_seq_push_ex": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.POINTER(VoUnitResult), C.c_void_p, C.c_int]),
    "vo_png_info": (C.c_int, [C.c_void_p, C.c_size_t, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "vo_png_decode": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]),
    "vo_png_last_error": (C.c_char_p, []),
    "vo_reader_open": (C.c_void_p, [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "vo_reader_next": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_int), C.POINTER(C.c_int),
                                 C.POINTER(C.c_size_t), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "vo_reader_error": (C.c_char_p, [C.c_void_p]),
    "vo_reader_close": (None, [C.c_void_p]),
    "vo_bgr_to_gray": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_size_t]),
    "vo_poses_load": (C.c_int, [C.c_char_p, C.c_void_p, C.c_int, C.POINTER(C.c_int)]),
    "vo_poses_save": (C.c_int, [C.c_char_p, C.c_void_p, C.c_int]),
    "vo_eval_segments": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int)]),
    "vo_eval_summary": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_float)]),
    "vo_pose_is_rotation": (C.c_int, [C.c_void_p]),
    "vo_pose_euler": (None, [C.c_void_p, C.c_void_p]),
    "vo_pose_integrate": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vo_pose_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "vo_seq_pose": (C.c_int, [C.c_void_p, C.c_void_p]),
    "vo_batch_fetch": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vo_mono_rotation": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_double, C.c_double, C.c_double, C.c_void_p,
                                   C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "vo_dist_unique_id": (C.c_int, [C.c_void_p]),
    "vo_dist_init": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int]),
    "vo_dist_gather_post": (C.c_int, [C.c_void_p, C.c_int, C.c_int]),
    "vo_dist_gather_wait": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int)]),
    "vo_batch_outputs": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_size_t)]),
    "vo_seq_begin_device": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(VoDImage), C.POINTER(VoDImage)]),
    "vo_seq_submit_device": (C.c_int, [C.c_void_p, C.POINTER(VoDImage), C.POINTER(VoDImage)]),
    "vo_batch_submit_device": (C.c_int, [C.c_void_p, C.POINTER(VoDUnit), C.c_int, C.c_int]),
    "vo_mseq_begin": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                C.c_int]),
    "vo_mseq_begin_ex": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_size_t, C.c_int, C.c_int]),
    "vo_mseq_begin_calib": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_size_t, C.c_int, C.c_int]),
    "vo_batch_calibrate": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vo_batch_params": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(VoParams)]),
    "vo_mseq_params": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(VoParams)]),
    "vo_mseq_begin_sized": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_int, C.c_int]),
    "vo_mseq_submit": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]),
    "vo_mseq_submit_sized": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]),
    "vo_mseq_open": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]),
    "vo_mseq_submit_start": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.POINTER(VoMseqStart)]),
    "vo_mseq_begin_device": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(VoDImage),
                                       C.POINTER(VoDImage), C.c_int]),
    "vo_mseq_submit_device": (C.c_int, [C.c_void_p, C.POINTER(VoDImage), C.POINTER(VoDImage), C.c_int, C.POINTER(VoMseqStart)]),
    "vo_mseq_wait": (C.c_int, [C.c_void_p, C.POINTER(VoUnitResult), C.c_void_p, C.c_void_p, C.c_int]),
    "vo_mseq_wait_mono": (C.c_int, [C.c_void_p, C.POINTER(VoUnitResult), C.c_void_p, C.POINTER(VoMonoResult), C.c_void_p,
                                    C.c_int, C.c_void_p, C.c_int]),
    "vo_mseq_wait_device": (C.c_int, [C.c_void_p, C.POINTER(VoMseqDResults)]),
    "vo_pose_step_device": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vo_mseq_pose": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p]),
    "vo_mseq_state": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int),
                                C.c_void_p]),
}

_lib = None


def load_library():
    """dlopen the in-tree CUDA library; raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: build it with `python -m visual_odom_b200.build` "
                "(there is no CPU fallback)")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name, None)
            if fn is None:
                continue            # reported by tests/test_abi.py
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class VoError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"vo_b200 error {code}: {msg}")
        self.code = code


class Context:
    """Owns one vo_ctx (one per GPU / host thread)."""

    def __init__(self, device=0, **params):
        self.lib = load_library()
        p = VoParams()
        self.lib.vo_default_params(C.byref(p))
        for k, v in params.items():
            if not hasattr(p, k):
                raise TypeError(f"unknown vo_params field {k}")
            setattr(p, k, v)
        self.params = p
        self.device = device
        self._stream = None           # the stream the context was last pointed at by the *_device calls
        self._bridge = None
        h = C.c_void_p()
        rc = self.lib.vo_create(device, C.byref(p), C.byref(h))
        self.h = h
        if rc != VO_OK:
            msg = self.lib.vo_last_error(h).decode() if h else "vo_create failed"
            if h:
                self.lib.vo_destroy(h)
            self.h = None
            raise VoError(rc, msg)

    def close(self):
        if getattr(self, "h", None):
            self.lib.vo_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, ok=(VO_OK,)):
        if rc not in ok:
            raise VoError(rc, self.lib.vo_last_error(self.h).decode())
        return rc

    # ---- plumbing --------------------------------------------------------------------------------
    def set_stream(self, cuda_stream_ptr):
        self._check(self.lib.vo_set_stream(self.h, C.c_void_p(cuda_stream_ptr)))
        self._stream = cuda_stream_ptr

    def sync(self):
        self._check(self.lib.vo_sync(self.h))

    def set_option(self, key, value):
        self._check(self.lib.vo_set_option(self.h, key.encode(), float(value)))

    def kernel_launches(self):
        return int(self.lib.vo_kernel_launches(self.h))

    def lk_kernel_time(self, reset=False):
        ms = C.c_double(); n = C.c_longlong()
        self._check(self.lib.vo_lk_kernel_time(self.h, C.byref(ms), C.byref(n), int(reset)))
        return ms.value, n.value

    # ---- single-call entry points (host buffers) -------------------------------------------------
    @staticmethod
    def _img(a):
        a = np.asarray(a)
        assert a.dtype == np.uint8 and a.ndim == 2, "images must be 2-D uint8 (CV_8UC1)"
        if a.strides[1] != 1:
            a = np.ascontiguousarray(a)
        return a

    def fast_detect(self, img, cap=None, with_response=False):
        img = self._img(img)
        h, w = img.shape
        cap = cap or self.params.max_features * 8
        out = np.zeros((cap, 2), np.float32)
        resp = np.zeros(cap, np.float32) if with_response else None
        n = C.c_int()
        self._check(self.lib.vo_fast_detect(self.h, _p(img), w, h, img.strides[0], _p(out), _p(resp), cap, C.byref(n)),
                    ok=(VO_OK, VO_E_CAPACITY))
        m = min(n.value, cap)
        return (out[:m], resp[:m], n.value) if with_response else (out[:m], n.value)

    def lk_track(self, prev, nxt, pts, want_err=True):
        prev = self._img(prev); nxt = self._img(nxt)
        assert prev.shape == nxt.shape and prev.strides == nxt.strides
        h, w = prev.shape
        pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
        n = len(pts)
        out = np.zeros((n, 2), np.float32); st = np.zeros(n, np.uint8)
        err = np.zeros(n, np.float32) if want_err else None
        self._check(self.lib.vo_lk_track(self.h, _p(prev), _p(nxt), w, h, prev.strides[0], _p(pts), n,
                                         _p(out), _p(st), _p(err)))
        return out, st, err

    def circular_match(self, l0, r0, l1, r1, pts, ages=None):
        imgs = [self._img(a) for a in (l0, r0, l1, r1)]
        assert all(a.shape == imgs[0].shape and a.strides == imgs[0].strides for a in imgs)
        h, w = imgs[0].shape
        pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
        n = len(pts)
        outs = [np.zeros((n, 2), np.float32) for _ in range(5)]
        status4 = np.zeros((4, n), np.uint8)
        raw4 = np.zeros((4, n, 2), np.float32)
        kept = np.zeros(n, np.int32)
        nk = C.c_int()
        ages_io = None if ages is None else np.ascontiguousarray(ages, np.int32).copy()
        self._check(self.lib.vo_circular_match(
            self.h, _p(imgs[0]), _p(imgs[1]), _p(imgs[2]), _p(imgs[3]), w, h, imgs[0].strides[0], _p(pts), n,
            _p(ages_io), _p(outs[0]), _p(outs[1]), _p(outs[2]), _p(outs[3]), _p(outs[4]), _p(status4), _p(raw4),
            _p(kept), C.byref(nk)))
        k = nk.value
        return {
            "l0": outs[0][:k], "r0": outs[1][:k], "l1": outs[2][:k], "r1": outs[3][:k], "l0_ret": outs[4][:k],
            "status4": status4, "raw4": raw4, "kept_idx": kept[:k],
            "ages": None if ages_io is None else ages_io[:k],
        }

    def triangulate(self, P_l, P_r, pts_l, pts_r):
        P_l = np.ascontiguousarray(P_l, np.float32).reshape(12); P_r = np.ascontiguousarray(P_r, np.float32).reshape(12)
        a = np.ascontiguousarray(pts_l, np.float32).reshape(-1, 2); b = np.ascontiguousarray(pts_r, np.float32).reshape(-1, 2)
        assert len(a) == len(b)
        X = np.zeros((len(a), 3), np.float32)
        self._check(self.lib.vo_triangulate(self.h, _p(P_l), _p(P_r), _p(a), _p(b), len(a), _p(X)))
        return X

    def triangulate_homogeneous(self, P_l, P_r, pts_l, pts_r):
        """(n, 4) float32: row i = column i of cv2.triangulatePoints' 4 x N output."""
        P_l = np.ascontiguousarray(P_l, np.float32).reshape(12); P_r = np.ascontiguousarray(P_r, np.float32).reshape(12)
        a = np.ascontiguousarray(pts_l, np.float32).reshape(-1, 2); b = np.ascontiguousarray(pts_r, np.float32).reshape(-1, 2)
        assert len(a) == len(b)
        X4 = np.zeros((len(a), 4), np.float32)
        self._check(self.lib.vo_triangulate_homogeneous(self.h, _p(P_l), _p(P_r), _p(a), _p(b), len(a), _p(X4)))
        return X4

    def mono_rotation(self, pts_t0, pts_t1, focal, pp):
        """findEssentialMat(RANSAC, 0.999, 1.0) + recoverPose: (R 3x3, inlier mask, RANSAC iterations)."""
        a = np.ascontiguousarray(pts_t0, np.float32).reshape(-1, 2); b = np.ascontiguousarray(pts_t1, np.float32).reshape(-1, 2)
        assert len(a) == len(b)
        R = np.zeros(9, np.float64); mask = np.zeros(max(len(a), 1), np.uint8)
        ni = C.c_int(0); it = C.c_int(0)
        self._check(self.lib.vo_mono_rotation(self.h, _p(a), _p(b), len(a), float(focal), float(pp[0]), float(pp[1]), _p(R), _p(mask),
                                              C.byref(ni), C.byref(it)))
        return R.reshape(3, 3), mask[:len(a)].astype(bool), it.value

    def pnp_ransac(self, X, x, K, rvec0=None, tvec0=None):
        X = np.ascontiguousarray(X, np.float32).reshape(-1, 3); x = np.ascontiguousarray(x, np.float32).reshape(-1, 2)
        assert len(X) == len(x)
        K = np.ascontiguousarray(K, np.float32).reshape(9)
        rvec = np.zeros(3) if rvec0 is None else np.ascontiguousarray(rvec0, np.float64).reshape(3).copy()
        tvec = np.zeros(3) if tvec0 is None else np.ascontiguousarray(tvec0, np.float64).reshape(3).copy()
        inl = np.zeros(max(len(X), 1), np.int32); n_in = C.c_int(); R = np.zeros(9); iters = C.c_int()
        rc = self.lib.vo_pnp_ransac(self.h, _p(X), _p(x), len(X), _p(K), _p(rvec), _p(tvec), _p(inl), C.byref(n_in),
                                    _p(R), C.byref(iters))
        self._check(rc)
        return {"rvec": rvec, "tvec": tvec, "R": R.reshape(3, 3), "inliers": inl[:n_in.value], "iters": iters.value}

    # ---- batched whole-path API ------------------------------------------------------------------
    def batch_configure(self, w, h, n_units, P_l, P_r):
        P_l = np.ascontiguousarray(P_l, np.float32).reshape(12); P_r = np.ascontiguousarray(P_r, np.float32).reshape(12)
        self._check(self.lib.vo_batch_configure(self.h, w, h, n_units, _p(P_l), _p(P_r)))
        self._batch_geom = (w, h, n_units)

    def batch_calibrate(self, first_unit, P_l, P_r):
        """Units [first_unit, first_unit + n) get their own calibrations: P_l / P_r of shape (n, 3, 4) (vo_batch_calibrate).
        Refused while submissions are in flight."""
        P_l = np.ascontiguousarray(P_l, np.float32); P_r = np.ascontiguousarray(P_r, np.float32)
        if P_l.ndim != 3 or P_l.shape[1:] != (3, 4) or P_r.shape != P_l.shape:
            raise ValueError(f"P_l / P_r must be (n, 3, 4), got {P_l.shape} / {P_r.shape}")
        self._check(self.lib.vo_batch_calibrate(self.h, first_unit, len(P_l), _p(P_l), _p(P_r)))

    def params_with(self, override=None):
        """A VoParams: the context's own (self.params) with the fields of the dict `override` (None: none) changed."""
        p = VoParams()
        C.memmove(C.byref(p), C.byref(self.params), C.sizeof(VoParams))
        for k, v in (override or {}).items():
            if not hasattr(p, k):
                raise TypeError(f"unknown vo_params field {k}")
            setattr(p, k, v)
        return p

    def _params_array(self, overrides):
        arr = (VoParams * len(overrides))()
        for i, o in enumerate(overrides):
            arr[i] = self.params_with(o)
        return arr

    def batch_params(self, first_unit, overrides):
        """Units [first_unit, first_unit + len(overrides)) get their own tracking parameters (vo_batch_params): each entry
        of `overrides` is a dict of the vo_params fields that differ from the context's, or None for the context's own.
        Refused while submissions are in flight."""
        if not overrides:
            raise ValueError("batch_params: no units")
        self._check(self.lib.vo_batch_params(self.h, first_unit, len(overrides), self._params_array(overrides)))

    def make_units(self, units):
        """units: list of dicts(l0,r0,l1,r1 uint8 HxW [, pts (n,2) f32 | n_select int] [, t_prev]).
        Returns (ctypes array, keep-alive list, pitch)."""
        arr = (VoUnit * len(units))()
        keep = []
        pitch = None
        for i, u in enumerate(units):
            imgs = [self._img(u[k]) for k in ("l0", "r0", "l1", "r1")]
            for a in imgs:
                assert a.shape == (self._batch_geom[1], self._batch_geom[0])
                pitch = pitch or a.strides[0]
                assert a.strides[0] == pitch
            keep.append(imgs)
            arr[i].l0, arr[i].r0, arr[i].l1, arr[i].r1 = (a.ctypes.data for a in imgs)
            if u.get("pts") is not None:
                pts = np.ascontiguousarray(u["pts"], np.float32).reshape(-1, 2)
                keep.append(pts)
                arr[i].pts = pts.ctypes.data
                arr[i].n_pts = len(pts)
            else:
                arr[i].pts = None
                arr[i].n_pts = int(u["n_select"])
            t = u.get("t_prev", (0.0, 0.0, 0.0))
            for k in range(3):
                arr[i].t_prev[k] = float(t[k])
        return arr, keep, pitch

    def batch_upload(self, arr, pitch):
        self._check(self.lib.vo_batch_upload(self.h, arr, len(arr), pitch))

    def batch_run(self):
        self._check(self.lib.vo_batch_run(self.h))

    def batch_download(self, n_units):
        res = (VoUnitResult * n_units)()
        self._check(self.lib.vo_batch_download(self.h, res, n_units))
        return [self._result_dict(r) for r in res]

    def frame_batch(self, arr, pitch):
        res = (VoUnitResult * len(arr))()
        self._check(self.lib.vo_frame_batch(self.h, arr, len(arr), pitch, res))
        return [self._result_dict(r) for r in res]

    def batch_submit(self, arr, first_unit, pitch, n_units=None):
        """Asynchronous upload + run + result staging of resident slots [first_unit, first_unit + len(arr));
        arr=None re-runs what is resident (n_units required)."""
        if arr is None:
            self._check(self.lib.vo_batch_submit(self.h, None, first_unit, n_units, pitch))
        else:
            self._check(self.lib.vo_batch_submit(self.h, arr, first_unit, len(arr), pitch))

    def batch_wait(self, first_unit, n_units, raw=False):
        """raw=True: the records as one numpy structured array (RESULT_DTYPE; fields are read as rec["n_valid"], rec["R"], ...)
        instead of a list of dicts."""
        res = (VoUnitResult * n_units)()
        self._check(self.lib.vo_batch_wait(self.h, first_unit, n_units, res))
        if raw:
            return np.frombuffer(res, dtype=RESULT_DTYPE)
        return [self._result_dict(r) for r in res]

    @staticmethod
    def _result_dict(r):
        return dict(n_features=r.n_features, n_detected=r.n_detected, n_tracked=r.n_tracked, n_valid=r.n_valid,
                    n_inliers=r.n_inliers, ransac_iters=r.ransac_iters, pnp_status=r.pnp_status,
                    rvec=np.array(r.rvec[:]), tvec=np.array(r.tvec[:]), R=np.array(r.R[:]).reshape(3, 3))

    @classmethod
    def _record(cls, r, cap, pts4=None, mono=None, mask=None, status=None):
        """A sequence frame's record as a dict: _result_dict's keys, with pts4 ((4, cap, 2) point lists) l0 / r0 / l1 / r1,
        with mono (a VoMonoResult) "mono" and the essential mask `mask` as "ess_mask", with status "status" (the first
        n_valid entries of the lists, none for a retired sequence)."""
        d = cls._result_dict(r)
        n = 0 if status == VO_MSEQ_RETIRED else min(d["n_valid"], cap)
        if status is not None:
            d["status"] = int(status)
        if pts4 is not None:
            d.update(l0=pts4[0, :n].copy(), r0=pts4[1, :n].copy(), l1=pts4[2, :n].copy(), r1=pts4[3, :n].copy())
        if mono is not None:
            d["mono"] = dict(status=mono.status, n_inliers=mono.n_inliers, ransac_iters=mono.ransac_iters, n_good=mono.n_good,
                             R=np.array(mono.R[:]).reshape(3, 3), t=np.array(mono.t[:]))
            d["ess_mask"] = mask[:n].astype(bool)
        return d

    @staticmethod
    def records_to_dicts(arr):
        """A RESULT_DTYPE array (batch_wait / dist_gather_wait with raw=True) as the list of dicts the other calls return."""
        ints = ("n_features", "n_detected", "n_tracked", "n_valid", "n_inliers", "ransac_iters", "pnp_status")
        return [dict({k: int(r[k]) for k in ints}, rvec=np.array(r["rvec"]), tvec=np.array(r["tvec"]), R=np.array(r["R"])) for r in arr]

    def batch_fetch(self, unit, res):
        nf, nv, ni = res["n_features"], res["n_valid"], res["n_inliers"]
        pts_in = np.zeros((max(nf, 1), 2), np.float32); pts4 = np.zeros((4, max(nv, 1), 2), np.float32)
        kept = np.zeros(max(nv, 1), np.int32); X = np.zeros((max(nv, 1), 3), np.float32); inl = np.zeros(max(ni, 1), np.int32)
        self._check(self.lib.vo_batch_fetch(self.h, unit, _p(pts_in), _p(pts4), _p(kept), _p(X), _p(inl)))
        return dict(pts_in=pts_in[:nf], l0=pts4[0, :nv], r0=pts4[1, :nv], l1=pts4[2, :nv], r1=pts4[3, :nv],
                    kept_idx=kept[:nv], X=X[:nv], inliers=inl[:ni])

    def batch_outputs(self, unit, res, into=None):
        """Point lists of a waited submission from the pinned block its single D2H filled (set_option("batch_outputs", 1)).
        `into` = preallocated dict(pts4, kept_idx, X, inliers) to avoid allocations in a timed loop."""
        nv, ni = res["n_valid"], res["n_inliers"]
        if into is None:
            into = dict(pts4=np.zeros((4, max(nv, 1), 2), np.float32), kept_idx=np.zeros(max(nv, 1), np.int32),
                        X=np.zeros((max(nv, 1), 3), np.float32), inliers=np.zeros(max(ni, 1), np.int32))
        nb = C.c_size_t(0)
        self._check(self.lib.vo_batch_outputs(self.h, unit, _p(into["pts4"]), _p(into["kept_idx"]), _p(into["X"]), _p(into["inliers"]),
                                              C.byref(nb)))
        flat = into["pts4"].reshape(-1, 2)            # the C side packs the four lists back to back (n_valid each)
        return dict(l0=flat[0:nv], r0=flat[nv:2 * nv], l1=flat[2 * nv:3 * nv], r1=flat[3 * nv:4 * nv], kept_idx=into["kept_idx"][:nv],
                    X=into["X"][:nv], inliers=into["inliers"][:ni], d2h_bytes=int(nb.value))

    # ---- multi-GPU record gather over NCCL (one process per GPU) -------------------------------------
    def dist_unique_id(self):
        buf = np.zeros(128, np.uint8)
        rc = self.lib.vo_dist_unique_id(_p(buf))
        if rc != VO_OK:
            raise VoError(rc, "vo_dist_unique_id: NCCL is not available on this host")
        return buf

    def dist_init(self, uid, rank, world):
        uid = np.ascontiguousarray(uid, np.uint8)
        assert uid.size == 128
        self._check(self.lib.vo_dist_init(self.h, _p(uid), int(rank), int(world)))
        self._dist_world = int(world)

    def dist_gather_post(self, first_unit, n_units):
        self._check(self.lib.vo_dist_gather_post(self.h, int(first_unit), int(n_units)))

    def dist_gather_wait(self, n_units, raw=False):
        """The oldest posted step's table (world x n_units records, rank-major).  raw=True: one numpy structured array
        (RESULT_DTYPE) instead of world x n_units dicts."""
        res = (VoUnitResult * (self._dist_world * n_units))()
        n = C.c_int(0)
        self._check(self.lib.vo_dist_gather_wait(self.h, res, len(res), C.byref(n)))
        if raw:
            return np.frombuffer(res, dtype=RESULT_DTYPE)[:n.value]
        return [self._result_dict(r) for r in res[:n.value]]

    # ---- streaming sequence mode -------------------------------------------------------------------
    def seq_begin(self, left0, right0, P_l, P_r):
        l = self._img(left0); r = self._img(right0)
        assert l.shape == r.shape and l.strides == r.strides
        P_l = np.ascontiguousarray(P_l, np.float32).reshape(12); P_r = np.ascontiguousarray(P_r, np.float32).reshape(12)
        self._check(self.lib.vo_seq_begin(self.h, l.shape[1], l.shape[0], _p(P_l), _p(P_r), _p(l), _p(r), l.strides[0]))

    def seq_push(self, left1, right1, pts_cap=4096, want_points=True, mono=False):
        """mono=True (a sequence begun with the option "mono_rotation"): submit + seq_wait(mono=True)."""
        l = self._img(left1); r = self._img(right1)
        if mono:
            self._check(self.lib.vo_seq_submit(self.h, _p(l), _p(r), l.strides[0], 1))
            return self.seq_wait(pts_cap, want_points, mono=True)
        res = VoUnitResult()
        pts4 = np.zeros((4, pts_cap, 2), np.float32) if want_points else None
        self._check(self.lib.vo_seq_push(self.h, _p(l), _p(r), l.strides[0], C.byref(res), _p(pts4), pts_cap if want_points else 0))
        return self._record(res, pts_cap, pts4)

    def seq_begin_bgr(self, left0, right0, P_l, P_r):
        """Colour (H x W x 3, BGR) inputs: converted on the device like cv::cvtColor(BGR2GRAY)."""
        l = np.ascontiguousarray(left0, np.uint8); r = np.ascontiguousarray(right0, np.uint8)
        assert l.ndim == 3 and l.shape[2] == 3 and r.shape == l.shape
        Pl = np.ascontiguousarray(P_l, np.float32); Pr = np.ascontiguousarray(P_r, np.float32)
        self._check(self.lib.vo_seq_begin_ex(self.h, l.shape[1], l.shape[0], _p(Pl), _p(Pr), _p(l), _p(r), l.strides[0], 3))

    def seq_push_bgr(self, left1, right1, pts_cap=4096):
        l = np.ascontiguousarray(left1, np.uint8); r = np.ascontiguousarray(right1, np.uint8)
        res = VoUnitResult()
        pts4 = np.zeros((4, pts_cap, 2), np.float32)
        self._check(self.lib.vo_seq_push_ex(self.h, _p(l), _p(r), l.strides[0], 3, C.byref(res), _p(pts4), pts_cap))
        return self._record(res, pts_cap, pts4)

    def seq_push_ptr(self, left_ptr, right_ptr, pitch, channels=1):
        """Raw host pointers (e.g. the pinned buffers a SequenceReader hands out); returns counts + pose only."""
        res = VoUnitResult()
        self._check(self.lib.vo_seq_push_ex(self.h, left_ptr, right_ptr, pitch, channels, C.byref(res), None, 0))
        return self._result_dict(res)

    def seq_begin_ptr(self, w, h, left_ptr, right_ptr, pitch, P_l, P_r, channels=1):
        Pl = np.ascontiguousarray(P_l, np.float32); Pr = np.ascontiguousarray(P_r, np.float32)
        self._check(self.lib.vo_seq_begin_ex(self.h, w, h, _p(Pl), _p(Pr), left_ptr, right_ptr, pitch, channels))

    def bgr_to_gray(self, bgr):
        """Stage-level entry point of the device gray conversion (H x W x 3 uint8 -> H x W uint8)."""
        a = np.ascontiguousarray(bgr, np.uint8)
        assert a.ndim == 3 and a.shape[2] == 3
        out = np.empty(a.shape[:2], np.uint8)
        self._check(self.lib.vo_bgr_to_gray(self.h, _p(a), a.strides[0], a.shape[1], a.shape[0], _p(out), out.strides[0]))
        return out

    def seq_submit(self, left1, right1):
        """Asynchronous push (gray H x W or BGR H x W x 3); at most two frames in flight. Keep the arrays alive."""
        l = np.asarray(left1); r = np.asarray(right1)
        ch = 3 if l.ndim == 3 else 1
        assert l.dtype == np.uint8 and l.shape == r.shape and l.strides[-1] == 1 and (ch == 1 or l.strides[1] == 3)
        self._check(self.lib.vo_seq_submit(self.h, _p(l), _p(r), l.strides[0], ch))

    def seq_submit_ptr(self, left_ptr, right_ptr, pitch, channels=1):
        self._check(self.lib.vo_seq_submit(self.h, left_ptr, right_ptr, pitch, channels))

    # ---- images already on the GPU (CUDA uint8 torch tensors (H, W), (H, W, 3) or (3, H, W)) ----------------------------
    # The calls run on torch.cuda.current_stream(): the images are read after the work already queued there, and work queued
    # there after the call is ordered after the library's last read of them, so a tensor may be overwritten or freed
    # stream-ordered at once (as after any PyTorch operation).  vo_set_stream synchronises the previous stream, so it is
    # called only when the current stream changes.  The legacy default stream cannot be captured into the library's CUDA
    # graphs: on it the context runs on a private stream that waits for the default stream before the call and is waited
    # for after it.
    def _device_image(self, t, order):
        import torch
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise TypeError("device images must be CUDA torch tensors (host images go through the host entry points)")
        if t.dtype != torch.uint8:
            raise TypeError(f"device images must be uint8, not {t.dtype}")
        if t.device.index != self.device:
            raise ValueError(f"image on {t.device}, the context on cuda:{self.device}")
        return image_descriptor(t.shape, t.stride(), t.data_ptr(), order)

    def _enter_stream(self):
        import torch
        cur = torch.cuda.current_stream(self.device)
        run = cur
        if cur.cuda_stream == 0:
            if self._bridge is None:
                self._bridge = torch.cuda.Stream(self.device)
            self._bridge.wait_stream(cur)
            run = self._bridge
        if run.cuda_stream != self._stream:
            self.set_stream(run.cuda_stream)
        return cur, run

    def _device_call(self, fn, *args):
        cur, run = self._enter_stream()
        try:
            self._check(fn(self.h, *args))
        finally:
            if run is not cur:
                cur.wait_stream(run)

    def seq_begin_device(self, left0, right0, P_l, P_r, order=None):
        (l, w, h), (r, wr, hr) = self._device_image(left0, order), self._device_image(right0, order)
        if (wr, hr) != (w, h):
            raise ValueError("left and right images differ in size")
        P_l = np.ascontiguousarray(P_l, np.float32).reshape(12); P_r = np.ascontiguousarray(P_r, np.float32).reshape(12)
        self._device_call(self.lib.vo_seq_begin_device, w, h, _p(P_l), _p(P_r), C.byref(l), C.byref(r))

    def seq_submit_device(self, left1, right1, order=None):
        """Asynchronous push of device images; results through seq_wait.  The tensors may be reused stream-ordered at once."""
        l, _, _ = self._device_image(left1, order)
        r, _, _ = self._device_image(right1, order)
        self._device_call(self.lib.vo_seq_submit_device, C.byref(l), C.byref(r))

    def seq_push_device(self, left1, right1, order=None, pts_cap=4096, want_points=True, mono=False):
        self.seq_submit_device(left1, right1, order)
        return self.seq_wait(pts_cap, want_points, mono=mono)

    def batch_submit_device(self, units, first_unit, order=None, n_units=None):
        """vo_batch_submit_device: units as for make_units, with CUDA tensors for l0, r0, l1, r1 (a colour unit may carry
        its own "order"); units=None re-runs what is resident (n_units required).  Results through batch_wait."""
        if units is None:
            self._device_call(self.lib.vo_batch_submit_device, None, first_unit, n_units)
            return
        arr = (VoDUnit * len(units))()
        keep = []
        for i, u in enumerate(units):
            for k in ("l0", "r0", "l1", "r1"):
                d, w, h = self._device_image(u[k], u.get("order", order))
                if (w, h) != tuple(self._batch_geom[:2]):
                    raise ValueError(f"unit {i} {k}: {w} x {h}, the batch is configured for {self._batch_geom[0]} x {self._batch_geom[1]}")
                setattr(arr[i], k, d)
            if u.get("pts") is not None:
                pts = np.ascontiguousarray(u["pts"], np.float32).reshape(-1, 2)
                keep.append(pts)
                arr[i].pts = pts.ctypes.data
                arr[i].n_pts = len(pts)
            else:
                arr[i].pts = None
                arr[i].n_pts = int(u["n_select"])
            t = u.get("t_prev", (0.0, 0.0, 0.0))
            for k in range(3):
                arr[i].t_prev[k] = float(t[k])
        self._device_call(self.lib.vo_batch_submit_device, arr, first_unit, len(units))

    def seq_wait(self, pts_cap=4096, want_points=True, mono=False):
        """mono=True: also "mono" (dict: status, n_inliers, ransac_iters, n_good, R 3x3, t) and "ess_mask" (bool, aligned
        with the point lists) of the same frame (vo_seq_wait_mono)."""
        res = VoUnitResult()
        pts4 = np.zeros((4, pts_cap, 2), np.float32) if want_points else None
        npts = pts_cap if want_points else 0
        if not mono:
            self._check(self.lib.vo_seq_wait(self.h, C.byref(res), _p(pts4), npts))
            return self._record(res, pts_cap, pts4)
        m = VoMonoResult()
        mask = np.zeros(pts_cap, np.uint8)
        self._check(self.lib.vo_seq_wait_mono(self.h, C.byref(res), C.byref(m), _p(mask), pts_cap, _p(pts4), npts))
        return self._record(res, pts_cap, pts4, m, mask)

    def seq_state(self, cap=1 << 17):
        pts = np.zeros((cap, 2), np.float32); ages = np.zeros(cap, np.int32); t = np.zeros(3)
        npts = C.c_int(); nages = C.c_int()
        self._check(self.lib.vo_seq_state(self.h, _p(pts), _p(ages), cap, C.byref(npts), C.byref(nages), _p(t)))
        return pts[:npts.value].copy(), ages[:nages.value].copy(), t

    def seq_pose(self):
        """frame_pose (4x4) integrated by seq_push since seq_begin (reference main.cpp:196-208)."""
        pose = np.zeros((4, 4))
        self._check(self.lib.vo_seq_pose(self.h, _p(pose)))
        return pose

    # ---- several sequences in lockstep (vo_mseq_*) --------------------------------------------------------------------
    @staticmethod
    def _pairs(lefts, rights, allow_none):
        """(left pointer table, right pointer table, pitch, channels, keep-alive, shape, shapes) of one image per sequence:
        gray H x W or BGR H x W x 3, one channel count for all; a pair's two images have one shape, the sequences may
        differ.  pitch is the packed row length when every shape is equal (None otherwise); shapes[q] is sequence q's
        shape (None for a None pair, which allow_none passes as two NULL pointers)."""
        if len(lefts) != len(rights):
            raise ValueError(f"{len(lefts)} left and {len(rights)} right images")
        n = len(lefts)
        lp, rp = (C.c_void_p * n)(), (C.c_void_p * n)()
        keep, shapes = [], [None] * n
        for q, (l, r) in enumerate(zip(lefts, rights)):
            if l is None and r is None and allow_none:
                continue
            if l is None or r is None:
                raise ValueError(f"sequence {q}: a pair needs both images (None, None retires a sequence)")
            l = np.asarray(l); r = np.asarray(r)
            if l.dtype != np.uint8 or l.ndim not in (2, 3) or (l.ndim == 3 and l.shape[2] != 3):
                raise ValueError(f"sequence {q}: images must be uint8 H x W (gray) or H x W x 3 (BGR)")
            l = np.ascontiguousarray(l); r = np.ascontiguousarray(r)
            if r.shape != l.shape:
                raise ValueError(f"sequence {q}: image shape {l.shape} / {r.shape}, expected one shape per pair")
            first = next((g for g in shapes if g is not None), None)
            if first is not None and len(first) != l.ndim:
                raise ValueError(f"sequence {q}: image shape {l.shape}, expected {'gray' if len(first) == 2 else 'BGR'} images")
            shapes[q] = l.shape
            keep += [l, r]
            lp[q], rp[q] = l.ctypes.data, r.ctypes.data
        live = [g for g in shapes if g is not None]
        if not live:
            return lp, rp, 0, 1, keep, None, shapes
        geom = live[0]
        ch = 1 if len(geom) == 2 else 3
        uniform = all(g == geom for g in live)
        return lp, rp, (geom[1] * ch if uniform else None), ch, keep, (geom if uniform else None), shapes

    def _mseq_begin(self, n, w, h, lp, rp, pitch, ch, P_l, P_r, mono_rotation):
        """P_l / P_r (3, 4): one calibration for every sequence (vo_mseq_begin_ex); (n, 3, 4): sequence q runs with
        P_l[q] / P_r[q] (vo_mseq_begin_calib).  w / h / pitch: one value for all, or one per sequence
        (vo_mseq_begin_sized, which takes the calibrations per sequence)."""
        P_l = np.ascontiguousarray(P_l, np.float32); P_r = np.ascontiguousarray(P_r, np.float32)
        flags = VO_MSEQ_MONO_ROTATION if mono_rotation else 0
        if any(np.ndim(v) > 0 for v in (w, h, pitch)):
            ws, hs, ps = (np.broadcast_to(np.asarray(v), (n,)) for v in (w, h, pitch))
            wa = np.ascontiguousarray(ws, np.int32); ha = np.ascontiguousarray(hs, np.int32)
            pa = np.ascontiguousarray(ps, np.uint64)
            if P_l.ndim == 2:
                P_l = np.ascontiguousarray(np.broadcast_to(P_l, (n, 3, 4)))
            if P_r.ndim == 2:
                P_r = np.ascontiguousarray(np.broadcast_to(P_r, (n, 3, 4)))
            if P_l.shape != (n, 3, 4) or P_r.shape != (n, 3, 4):
                raise ValueError(f"per-sequence calibrations must be ({n}, 3, 4), got {P_l.shape} / {P_r.shape}")
            self._check(self.lib.vo_mseq_begin_sized(self.h, n, _p(wa), _p(ha), _p(P_l), _p(P_r), lp, rp, _p(pa), ch, flags))
            self._mseq_mono = bool(mono_rotation)
            self._mseq_n, self._mseq_pitch = n, pa.copy()
            self._mseq_sizes = [(int(a), int(b)) for a, b in zip(ha, wa)]
            self._mseq_keep = [None, None]
            return
        if P_l.ndim == 3 or P_r.ndim == 3:
            if P_l.shape != (n, 3, 4) or P_r.shape != (n, 3, 4):
                raise ValueError(f"per-sequence calibrations must be ({n}, 3, 4), got {P_l.shape} / {P_r.shape}")
            self._check(self.lib.vo_mseq_begin_calib(self.h, n, w, h, _p(P_l), _p(P_r), lp, rp, pitch, ch, flags))
        else:
            P_l = P_l.reshape(12); P_r = P_r.reshape(12)
            self._check(self.lib.vo_mseq_begin_ex(self.h, n, w, h, _p(P_l), _p(P_r), lp, rp, pitch, ch, flags))
        self._mseq_n, self._mseq_pitch = n, pitch
        self._mseq_mono = bool(mono_rotation)
        self._mseq_sizes = [(int(h), int(w))] * n
        self._mseq_keep = [None, None]

    def mseq_begin(self, lefts, rights, P_l, P_r, mono_rotation=False):
        """Start len(lefts) sequences from their first stereo pairs.  The sequences may differ in image size (gray or BGR
        for all): each then runs at its own size (vo_mseq_begin_sized).  P_l / P_r: (3, 4) for one calibration, or
        (n_seq, 3, 4) for one per sequence.  mono_rotation=True: every sequence runs trackingFrame2Frame(mono_rotation =
        true) (flag VO_MSEQ_MONO_ROTATION; see mseq_wait(mono=True))."""
        lp, rp, pitch, ch, keep, geom, shapes = self._pairs(lefts, rights, False)
        if geom is None and shapes and shapes[0] is not None:         # several sizes
            w = [g[1] for g in shapes]; h = [g[0] for g in shapes]
            pitch = [g[1] * ch for g in shapes]
        else:
            h, w = (geom or (0, 0))[:2]
        self._mseq_begin(len(lefts), w, h, lp, rp, pitch, ch, P_l, P_r, mono_rotation)

    def mseq_begin_ptr(self, w, h, left_ptrs, right_ptrs, pitch, P_l, P_r, channels=1, mono_rotation=False):
        """Raw host pointers, one pair per sequence (e.g. the pinned buffers of one SequenceReader each); P_l / P_r as for
        mseq_begin.  w / h / pitch: one value for every sequence, or a sequence of one per sequence (vo_mseq_begin_sized)."""
        n = len(left_ptrs)
        lp, rp = (C.c_void_p * n)(*left_ptrs), (C.c_void_p * n)(*right_ptrs)
        self._mseq_begin(n, w, h, lp, rp, pitch, channels, P_l, P_r, mono_rotation)

    def mseq_params(self, first_slot, overrides):
        """Slots [first_slot, first_slot + len(overrides)) get their own tracking parameters (vo_mseq_params), read by the
        next begin, open or start of each slot: each entry of `overrides` is a dict of the vo_params fields that differ
        from the context's, or None for the context's own.  Host state only: allowed while frames are in flight."""
        if not overrides:
            raise ValueError("mseq_params: no slots")
        self._check(self.lib.vo_mseq_params(self.h, first_slot, len(overrides), self._params_array(overrides)))

    def mseq_open(self, n_slots, max_w, max_h, mono_rotation=False, device_results=False):
        """n_slots empty slots for sequences of any size inside max_w x max_h with that size's pyramid depth
        (vo_mseq_open); sequences come in through mseq_submit(start=...).  mono_rotation=True: every sequence started in
        the run runs trackingFrame2Frame(mono_rotation = true).  device_results=True: the run takes its frames through
        mseq_submit_device and returns its results through mseq_wait_device (VO_MSEQ_DEVICE_RESULTS)."""
        flags = (VO_MSEQ_MONO_ROTATION if mono_rotation else 0) | (VO_MSEQ_DEVICE_RESULTS if device_results else 0)
        self._check(self.lib.vo_mseq_open(self.h, int(n_slots), int(max_w), int(max_h), flags))
        self._mseq_mono = bool(mono_rotation)
        self._mseq_n, self._mseq_pitch = int(n_slots), np.zeros(int(n_slots), np.uint64)
        self._mseq_sizes = [None] * int(n_slots)
        self._mseq_keep = [None, None]

    @staticmethod
    def _starts(start):
        """{slot: (w, h, P_l, P_r)} as a vo_mseq_start array and its length."""
        arr = (VoMseqStart * max(len(start), 1))()
        for s, (q, (w, h, P_l, P_r)) in zip(arr, start.items()):
            s.slot, s.w, s.h = int(q), int(w), int(h)
            s.P_l[:] = np.asarray(P_l, np.float32).reshape(12).tolist()
            s.P_r[:] = np.asarray(P_r, np.float32).reshape(12).tolist()
        return arr, len(start)

    def mseq_submit_ptr(self, left_ptrs, right_ptrs, pitch, channels=1, start=None):
        """Raw host pointers; None in both lists retires that sequence.  The memory must stay valid until the wait.
        pitch: one row pitch for every image, or a sequence of one per sequence (vo_mseq_submit_sized).
        start = {slot: (w, h, P_l, P_r)}: those slots' pairs are the first pairs of new sequences (vo_mseq_submit_start)."""
        n = len(left_ptrs)
        lp, rp = (C.c_void_p * n)(*left_ptrs), (C.c_void_p * n)(*right_ptrs)
        if start:
            pa = np.ascontiguousarray(np.broadcast_to(np.asarray(pitch), (n,)), np.uint64)
            arr, ns = self._starts(start)
            self._check(self.lib.vo_mseq_submit_start(self.h, lp, rp, _p(pa), channels, ns, arr))
        elif np.ndim(pitch) > 0:
            pa = np.ascontiguousarray(np.broadcast_to(np.asarray(pitch), (n,)), np.uint64)
            self._check(self.lib.vo_mseq_submit_sized(self.h, lp, rp, _p(pa), channels))
        else:
            self._check(self.lib.vo_mseq_submit(self.h, lp, rp, pitch, channels))

    def mseq_submit(self, lefts, rights, start=None):
        """Asynchronous: one frame of every sequence; a (None, None) pair retires that sequence.  At most two submissions
        in flight.  The arrays are kept alive by the context until their submission has been waited for.
        start = {slot: (P_l, P_r)}: those slots' pairs are the first pairs of new sequences with these matrices, at the
        pairs' sizes (vo_mseq_submit_start; the wait of this submission reports VO_MSEQ_STARTED for them)."""
        lp, rp, pitch, ch, keep, geom, shapes = self._pairs(lefts, rights, True)
        if len(lefts) != getattr(self, "_mseq_n", len(lefts)):
            raise ValueError(f"{len(lefts)} pairs for {self._mseq_n} sequences")
        start = dict(start or {})
        for q in start:
            if not 0 <= q < len(shapes) or shapes[q] is None:
                raise ValueError(f"slot {q}: a start needs its first pair")
        sized = np.ndim(self._mseq_pitch) > 0
        if sized or start:                          # several sizes or starts: one packed pitch per live pair
            for q, g in enumerate(shapes):
                if sized and g is not None and q not in start and self._mseq_sizes[q] is not None \
                        and tuple(g[:2]) != self._mseq_sizes[q]:
                    raise ValueError(f"sequence {q}: image shape {g}, the sequence is {self._mseq_sizes[q]}")
            pa = np.array([g[1] * ch if g is not None else 0 for g in shapes], np.uint64)
            if start:
                arr, ns = self._starts({q: (shapes[q][1], shapes[q][0], P[0], P[1]) for q, P in start.items()})
                self._check(self.lib.vo_mseq_submit_start(self.h, lp, rp, _p(pa), ch, ns, arr))
                if sized:
                    for q in start:
                        self._mseq_sizes[q] = tuple(shapes[q][:2])
            else:
                self._check(self.lib.vo_mseq_submit_sized(self.h, lp, rp, _p(pa), ch))
        else:
            if pitch is None:
                raise ValueError("the sequences were begun with one image size: every pair needs that shape")
            # with every sequence retired no image is read: the pitch of the first pairs passes the width check
            self._check(self.lib.vo_mseq_submit(self.h, lp, rp, pitch or self._mseq_pitch, ch))
        self._mseq_keep = [self._mseq_keep[1], keep]

    # ---- several sequences from images already on the GPU (vo_mseq_begin_device / vo_mseq_submit_device) ------------------
    def _device_pairs(self, lefts, rights, order, n, allow_none):
        """(left descriptor table, right descriptor table, sizes) of one pair of CUDA uint8 tensors per sequence, as
        _device_image reads them; sizes[q] = (h, w) of sequence q's pair, None for a (None, None) pair (allow_none: NULL
        descriptors, which retire the sequence).  order: one string for every colour pair, or one per sequence."""
        if len(lefts) != n or len(rights) != n:
            raise ValueError(f"{len(lefts)} left and {len(rights)} right images for {n} sequences")
        orders = [order] * n if order is None or isinstance(order, str) else list(order)
        if len(orders) != n:
            raise ValueError(f"{len(orders)} orders for {n} sequences")
        lt, rt = (VoDImage * n)(), (VoDImage * n)()
        sizes = [None] * n
        for q, (l, r) in enumerate(zip(lefts, rights)):
            if l is None and r is None and allow_none:
                continue
            if l is None or r is None:
                raise ValueError(f"sequence {q}: a pair needs both images (None, None retires a sequence)")
            (dl, w, h), (dr, wr, hr) = self._device_image(l, orders[q]), self._device_image(r, orders[q])
            if (wr, hr) != (w, h):
                raise ValueError(f"sequence {q}: left image {w} x {h}, right image {wr} x {hr}")
            lt[q], rt[q], sizes[q] = dl, dr, (h, w)
        return lt, rt, sizes

    def mseq_begin_device(self, lefts, rights, P_l, P_r, order=None, mono_rotation=False, device_results=False):
        """mseq_begin from CUDA uint8 tensors (H, W), (H, W, 3) or (3, H, W), one pair per sequence, each sequence at its
        pair's size and in its own layout (vo_mseq_begin_device; synchronous).  order: "bgr" / "rgb" for colour pairs, one
        string or one per sequence.  P_l / P_r: (3, 4) for one calibration, or (n_seq, 3, 4).  device_results=True: results
        through mseq_wait_device only (VO_MSEQ_DEVICE_RESULTS)."""
        n = len(lefts)
        lt, rt, sizes = self._device_pairs(lefts, rights, order, n, False)
        P_l = np.ascontiguousarray(np.broadcast_to(np.asarray(P_l, np.float32), (n, 3, 4)))
        P_r = np.ascontiguousarray(np.broadcast_to(np.asarray(P_r, np.float32), (n, 3, 4)))
        wa = np.array([g[1] for g in sizes], np.int32); ha = np.array([g[0] for g in sizes], np.int32)
        flags = (VO_MSEQ_MONO_ROTATION if mono_rotation else 0) | (VO_MSEQ_DEVICE_RESULTS if device_results else 0)
        self._device_call(self.lib.vo_mseq_begin_device, n, _p(wa), _p(ha), _p(P_l), _p(P_r), lt, rt, flags)
        self._mseq_mono = bool(mono_rotation)
        # host submissions may follow: the pitch state mseq_begin leaves for these sizes
        uniform = all(g == sizes[0] for g in sizes)
        self._mseq_n, self._mseq_pitch = n, (int(wa[0]) if uniform else wa.astype(np.uint64))
        self._mseq_sizes = list(sizes)
        self._mseq_keep = [None, None]

    def mseq_submit_device(self, lefts, rights, start=None, order=None):
        """mseq_submit from CUDA uint8 tensors (vo_mseq_submit_device): one frame of every sequence, a (None, None) pair
        retires that sequence; start = {slot: (P_l, P_r)} starts new sequences at their pairs' sizes.  Each pair must have
        its sequence's size.  The tensors may be overwritten or freed stream-ordered as soon as the call returns."""
        n = self._mseq_n
        lt, rt, sizes = self._device_pairs(lefts, rights, order, n, True)
        start = dict(start or {})
        for q in start:
            if not 0 <= q < n or sizes[q] is None:
                raise ValueError(f"slot {q}: a start needs its first pair")
        known = getattr(self, "_mseq_sizes", [None] * n)
        for q, g in enumerate(sizes):
            if g is not None and q not in start and known[q] is not None and g != known[q]:
                raise ValueError(f"sequence {q}: image size {g[1]} x {g[0]}, the sequence is {known[q][1]} x {known[q][0]}")
        arr, ns = self._starts({q: (sizes[q][1], sizes[q][0], P[0], P[1]) for q, P in start.items()}) if start else (None, 0)
        self._device_call(self.lib.vo_mseq_submit_device, lt, rt, ns, arr)
        for q in start:
            self._mseq_sizes[q] = sizes[q]
        self._mseq_keep = [self._mseq_keep[1], None]        # a host submission still in flight keeps its arrays

    def mseq_wait(self, pts_cap=4096, want_points=True, mono=False):
        """The oldest submission: one dict per sequence with seq_wait's keys plus "status" (VO_OK, VO_E_CAPACITY or
        VO_MSEQ_RETIRED).  mono=True (sequences begun with mono_rotation=True): also "mono" and "ess_mask" per sequence, as
        seq_wait(mono=True) gives them (vo_mseq_wait_mono; a retired sequence's "mono" is zeroed, its mask empty)."""
        n = self._mseq_n
        res = (VoUnitResult * n)()
        st = np.zeros(n, np.int32)
        pts4 = np.zeros((n, 4, pts_cap, 2), np.float32) if want_points else None
        npts = pts_cap if want_points else 0
        if mono:
            ms = (VoMonoResult * n)()
            mask = np.zeros((n, pts_cap), np.uint8)
            self._check(self.lib.vo_mseq_wait_mono(self.h, res, _p(st), ms, _p(mask), pts_cap, _p(pts4), npts), ok=(VO_OK, VO_E_CAPACITY))
        else:
            self._check(self.lib.vo_mseq_wait(self.h, res, _p(st), _p(pts4), npts), ok=(VO_OK, VO_E_CAPACITY))
        return [self._record(res[q], pts_cap, None if pts4 is None else pts4[q], ms[q] if mono else None,
                             mask[q] if mono else None, st[q]) for q in range(n)]

    def mseq_dresults_alloc(self, pts_cap=4096, points=True, points3d=True, inliers=True, mono=False):
        """The CUDA tensors mseq_wait_device writes for the run's n_seq sequences (pass them back as out= to reuse them):
        "records" (n, 19) float64 holds vo_unit_result records, viewed as "counts" (n, 7) int32 (n_features, n_detected,
        n_tracked, n_valid, n_inliers, ransac_iters, pnp_status), "rvec" / "tvec" (n, 3) and "R" (n, 3, 3); "status" (n,)
        int32; "frame_pose" (n, 4, 4) float64; "pts4" (n, 4, pts_cap, 2) float32 (L0, R0, L1, R1); "points3d"
        (n, pts_cap, 3) float32; "inliers" (n, pts_cap) int32; with mono, "mono_raw" (n, 14) float64 holds vo_mono_result,
        viewed as "mono_counts" (n, 4) int32 (status, n_inliers, ransac_iters, n_good), "mono_R" (n, 3, 3), "mono_t" (n, 3),
        and "ess_mask" (n, pts_cap) uint8."""
        import torch
        n, dev = self._mseq_n, torch.device("cuda", self.device)
        lists = points or points3d or inliers or mono
        if lists and (not isinstance(pts_cap, (int, np.integer)) or pts_cap <= 0):
            raise ValueError(f"pts_cap = {pts_cap!r}: point outputs need pts_cap > 0")
        rec = torch.zeros((n, 19), dtype=torch.float64, device=dev)
        out = dict(records=rec, counts=rec[:, :4].view(torch.int32)[:, :7], rvec=rec[:, 4:7], tvec=rec[:, 7:10],
                   R=rec[:, 10:19].view(n, 3, 3), status=torch.zeros(n, dtype=torch.int32, device=dev),
                   frame_pose=torch.zeros((n, 4, 4), dtype=torch.float64, device=dev), pts_cap=int(pts_cap) if lists else 0)
        if points:
            out["pts4"] = torch.zeros((n, 4, pts_cap, 2), dtype=torch.float32, device=dev)
        if points3d:
            out["points3d"] = torch.zeros((n, pts_cap, 3), dtype=torch.float32, device=dev)
        if inliers:
            out["inliers"] = torch.zeros((n, pts_cap), dtype=torch.int32, device=dev)
        if mono:
            m = torch.zeros((n, 14), dtype=torch.float64, device=dev)
            out.update(mono_raw=m, mono_counts=m[:, :2].view(torch.int32), mono_R=m[:, 2:11].view(n, 3, 3), mono_t=m[:, 11:14],
                       ess_mask=torch.zeros((n, pts_cap), dtype=torch.uint8, device=dev))
        return out

    _DRES_SHAPES = {"records": ("float64", (19,)), "status": ("int32", ()), "frame_pose": ("float64", (4, 4)),
                    "pts4": ("float32", (4, None, 2)), "points3d": ("float32", (None, 3)), "inliers": ("int32", (None,)),
                    "mono_raw": ("float64", (14,)), "ess_mask": ("uint8", (None,))}

    def mseq_wait_device(self, pts_cap=4096, points=True, points3d=True, inliers=True, out=None):
        """Retire the oldest submission of a run begun with device_results=True without blocking the host
        (vo_mseq_wait_device): one kernel on torch.cuda.current_stream() writes every sequence's results into CUDA tensors,
        which work queued on that stream afterwards may read at once.  Returns the dict of mseq_dresults_alloc (with
        "mono_*" and "ess_mask" in runs begun with mono_rotation=True); out= such a dict, which is filled in place, so a
        loop allocates nothing.  Only the first n_valid entries of a sequence's point lists (inliers: n_inliers) are
        defined."""
        mono = bool(getattr(self, "_mseq_mono", False))
        if out is None:
            out = self.mseq_dresults_alloc(pts_cap, points, points3d, inliers, mono)
        else:
            self._check_dresults(out)
        r = VoMseqDResults()
        r.pts_cap = int(out.get("pts_cap", 0))
        for f, k in (("status", "status"), ("records", "records"), ("frame_pose", "frame_pose"), ("pts4", "pts4"),
                     ("points3d", "points3d"), ("inliers", "inliers"), ("mono", "mono_raw"), ("ess_mask", "ess_mask")):
            t = out.get(k)
            setattr(r, f, None if t is None else t.data_ptr())
        self._device_call(self.lib.vo_mseq_wait_device, C.byref(r))
        return out

    def _check_dresults(self, out):
        """out= of mseq_wait_device: CUDA tensors on the context's GPU, contiguous, of the run's sequence count, the
        dtypes mseq_dresults_alloc gives and one pts_cap."""
        import torch
        n = self._mseq_n
        cap = out.get("pts_cap", 0)
        for k, (dt, tail) in self._DRES_SHAPES.items():
            t = out.get(k)
            if t is None:
                continue
            want = (n,) + tuple(cap if d is None else d for d in tail)
            if not isinstance(t, torch.Tensor):
                raise TypeError(f"out[{k!r}] must be a CUDA tensor on cuda:{self.device}")
            if str(t.dtype) != "torch." + dt or tuple(t.shape) != want or not t.is_contiguous():
                raise ValueError(f"out[{k!r}]: {tuple(t.shape)} {t.dtype}, expected a contiguous {want} {dt}")
            if not t.is_cuda or t.device.index != self.device:
                raise TypeError(f"out[{k!r}] must be a CUDA tensor on cuda:{self.device}")

    def pose_step_device(self, frame_pose, R, t):
        """vo_pose_step of n frames by the device function vo_mseq_wait_device integrates with (vo_pose_step_device):
        frame_pose (n, 4, 4), R (n, 3, 3), t (n, 3) -> (new poses, return codes)."""
        pose = np.array(frame_pose, np.float64).reshape(-1, 16).copy()
        n = len(pose)
        R = np.ascontiguousarray(R, np.float64).reshape(n, 9); t = np.ascontiguousarray(t, np.float64).reshape(n, 3)
        rc = np.zeros(n, np.int32)
        self._check(self.lib.vo_pose_step_device(self.h, n, _p(pose), _p(R), _p(t), _p(rc)))
        return pose.reshape(n, 4, 4), rc

    def mseq_pose(self, q):
        pose = np.zeros((4, 4))
        self._check(self.lib.vo_mseq_pose(self.h, int(q), _p(pose)))
        return pose

    def mseq_state(self, q, cap=1 << 17):
        pts = np.zeros((cap, 2), np.float32); ages = np.zeros(cap, np.int32); t = np.zeros(3)
        npts = C.c_int(); nages = C.c_int()
        self._check(self.lib.vo_mseq_state(self.h, int(q), _p(pts), _p(ages), cap, C.byref(npts), C.byref(nages), _p(t)))
        return pts[:npts.value].copy(), ages[:nages.value].copy(), t


# ---- host-only pose bookkeeping (SURVEY.md 8f row N2; no GPU needed) ------------------------------------------------
def pose_euler(R):
    R = np.ascontiguousarray(R, np.float64); e = np.zeros(3, np.float32)
    load_library().vo_pose_euler(_p(R), _p(e))
    return e


def pose_is_rotation(R):
    R = np.ascontiguousarray(R, np.float64)
    return bool(load_library().vo_pose_is_rotation(_p(R)))


def pose_integrate(frame_pose, R, t):
    """integrateOdometryStereo: returns (new_pose, rigid_inv, advanced)."""
    pose = np.array(frame_pose, np.float64).reshape(4, 4).copy(); inv = np.zeros((4, 4))
    R = np.ascontiguousarray(R, np.float64); t = np.ascontiguousarray(t, np.float64).reshape(3)
    rc = load_library().vo_pose_integrate(_p(pose), _p(R), _p(t), _p(inv))
    if rc < 0:
        raise RuntimeError("vo_pose_integrate: singular transformation")
    return pose, inv, bool(rc)


def pose_step(frame_pose, R, t):
    """Euler gate + integration (main.cpp:196-208): returns (new_pose, advanced)."""
    pose = np.array(frame_pose, np.float64).reshape(4, 4).copy()
    R = np.ascontiguousarray(R, np.float64); t = np.ascontiguousarray(t, np.float64).reshape(3)
    rc = load_library().vo_pose_step(_p(pose), _p(R), _p(t))
    if rc < 0:
        raise RuntimeError("vo_pose_step: singular transformation")
    return pose, bool(rc)


# ---- image ingest (SURVEY.md 8f row N3): host-side PNG decode + prefetching KITTI-layout reader ----------------------
def png_info(data):
    buf = np.frombuffer(data, np.uint8)
    w = C.c_int(); h = C.c_int(); ct = C.c_int(); bd = C.c_int()
    lib = load_library()
    if lib.vo_png_info(_p(buf), buf.size, C.byref(w), C.byref(h), C.byref(ct), C.byref(bd)) != 0:
        raise RuntimeError(lib.vo_png_last_error().decode())
    return w.value, h.value, ct.value, bd.value


def png_decode(data, want_bgr=True, want_gray=True):
    """bytes of one PNG -> (bgr HxWx3 | None, gray HxW | None): imread(IMREAD_COLOR) and cvtColor(BGR2GRAY) of it."""
    buf = np.frombuffer(data, np.uint8)
    w, h, _, _ = png_info(data)
    bgr = np.empty((h, w, 3), np.uint8) if want_bgr else None
    gray = np.empty((h, w), np.uint8) if want_gray else None
    lib = load_library()
    rc = lib.vo_png_decode(_p(buf), buf.size, _p(bgr) if want_bgr else None, 3 * w, _p(gray) if want_gray else None, w)
    if rc != 0:
        raise RuntimeError(lib.vo_png_last_error().decode())
    return bgr, gray


class SequenceReader:
    """<dir>/image_0/%06d.png + <dir>/image_1/%06d.png decoded ahead on worker threads into pinned buffers."""

    def __init__(self, sequence_dir, first_frame, n_frames, threads=4, depth=4, force_channels=0):
        self.lib = load_library()
        self.h = self.lib.vo_reader_open(str(sequence_dir).encode(), first_frame, n_frames, threads, depth, force_channels)
        if not self.h:
            raise RuntimeError("vo_reader_open: " + self.lib.vo_png_last_error().decode())
        self.n_frames = n_frames

    def next_ptr(self):
        """(left_ptr, right_ptr, w, h, pitch, channels, frame_id); pointers valid until the second following call."""
        l = C.c_void_p(); r = C.c_void_p(); w = C.c_int(); h = C.c_int(); p = C.c_size_t(); ch = C.c_int(); fid = C.c_int()
        rc = self.lib.vo_reader_next(self.h, C.byref(l), C.byref(r), C.byref(w), C.byref(h), C.byref(p), C.byref(ch), C.byref(fid))
        if rc != 0:
            raise RuntimeError("vo_reader_next: " + self.lib.vo_reader_error(self.h).decode())
        return l.value, r.value, w.value, h.value, p.value, ch.value, fid.value

    def next(self):
        """Copies of the frame's two images as numpy arrays (H x W or H x W x 3) + frame id."""
        l, r, w, h, p, ch, fid = self.next_ptr()
        shape = (h, w) if ch == 1 else (h, w, 3)
        n = h * p
        la = np.ctypeslib.as_array((C.c_uint8 * n).from_address(l)).reshape(shape).copy()
        ra = np.ctypeslib.as_array((C.c_uint8 * n).from_address(r)).reshape(shape).copy()
        return la, ra, fid

    def close(self):
        if self.h:
            self.lib.vo_reader_close(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ---- KITTI accuracy evaluation (SURVEY.md 8f row N4; host-only) -------------------------------------------------------
SEGMENT_DTYPE = np.dtype([("first_frame", np.int32), ("r_err", np.float32), ("t_err", np.float32), ("len", np.float32),
                          ("speed", np.float32)])


def poses_load(path):
    lib = load_library()
    n = C.c_int()
    if lib.vo_poses_load(str(path).encode(), None, 0, C.byref(n)) != 0:
        raise RuntimeError(f"cannot read poses from {path}")
    out = np.zeros((n.value, 12))
    if n.value:
        lib.vo_poses_load(str(path).encode(), _p(out), n.value, C.byref(n))
    return out


def poses_save(path, poses):
    p = np.ascontiguousarray(np.asarray(poses, np.float64).reshape(len(poses), -1)[:, :12])
    if load_library().vo_poses_save(str(path).encode(), _p(p), len(p)) != 0:
        raise RuntimeError(f"cannot write poses to {path}")


def eval_segments(gt, est, lengths=None, step=10):
    """KITTI segment errors of `est` against `gt` (n x 12 or n x 4 x 4 poses) -> (segments, t_err_avg, r_err_avg)."""
    def rows(a):
        a = np.asarray(a, np.float64)
        return np.ascontiguousarray(a.reshape(len(a), -1)[:, :12])
    g, e = rows(gt), rows(est)
    assert g.shape == e.shape
    lib = load_library()
    L = np.ascontiguousarray(lengths, np.float32) if lengths is not None else None
    n = C.c_int()
    args = (_p(g), _p(e), len(g), _p(L) if L is not None else None, len(L) if L is not None else 0, step)
    if lib.vo_eval_segments(*args, None, 0, C.byref(n)) != 0:
        raise RuntimeError("vo_eval_segments failed (singular pose?)")
    seg = np.zeros(n.value, SEGMENT_DTYPE)
    if n.value == 0:
        return seg, float("nan"), float("nan")
    lib.vo_eval_segments(*args, _p(seg), n.value, C.byref(n))
    t = C.c_float(); r = C.c_float()
    lib.vo_eval_summary(_p(seg), n.value, C.byref(t), C.byref(r))
    return seg, t.value, r.value
