"""
oracle/cref.py -- TEST INFRASTRUCTURE ONLY.  ctypes access to the plain-C restatements
(oracle/lk_ref.c, oracle/fast_ref.c -> oracle/_build/liboracle.so, built by
visual_odom_b200/build.py:build_oracle or __graft_entry__.build()).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module.  It is the checker, never the product.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_build", "liboracle.so")
_lib = None

# lk_track's event log (lk_ref.c: lk_event_t and the LK_EV_* kinds)
LK_EVENT = np.dtype([("pt", "<i4"), ("level", "<i4"), ("iter", "<i4"), ("kind", "<i4"),
                     ("min_eig", "<f4"), ("D", "<f4"), ("dx", "<f4"), ("dy", "<f4"), ("sdx", "<f4"), ("sdy", "<f4"),
                     ("ipx", "<i4"), ("ipy", "<i4"), ("inx", "<i4"), ("iny", "<i4"),
                     ("d2", "<f8"), ("d2f", "<f4"), ("pad_", "<i4"), ("sabs", "<i8", (10,)),
                     ("pos", "<i8", (10,)), ("neg", "<i8", (10,)), ("total", "<i8", (10,)),
                     ("maxpre", "<i8", (10,)), ("maxadd", "<i8", (10,)), ("fchain", "<f4", (10,))])
EV_ITER, EV_EPS, EV_HALF, EV_CAP, EV_JOUT, EV_SETUP, EV_REJECT, EV_IOUT, EV_FINAL = range(9)

# lk_set_sum_mode (lk_ref.c: LK_SUM_*).  SUM_CV2 is the pinned order; SUM_KERNEL is k_lk_ring's exact-path vote and
# combination (equal to SUM_CV2 on every input); SUM_M1..SUM_M6 are wrong votes or orders.  SUM_WIN is k_lk_win's b
# chains (equal to SUM_CV2); SUM_TAILCOL, SUM_SIMD4, SUM_ADJ and SUM_COMBINE are wrong orders of them (vote-free)
SUM_CV2, SUM_SEQ, SUM_PAIRS, SUM_SCALAR = 0, 1, 2, 9
SUM_KERNEL, SUM_M1, SUM_M2, SUM_M3, SUM_M4, SUM_M5, SUM_M6 = range(10, 17)
SUM_WIN, SUM_TAILCOL, SUM_SIMD4, SUM_ADJ, SUM_COMBINE = range(17, 22)


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} missing: run `python -m visual_odom_b200.build`")
        L = C.CDLL(LIB_PATH)
        L.lk_pyr_build.restype = C.c_void_p
        L.lk_pyr_build.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
        L.lk_pyr_free.argtypes = [C.c_void_p]
        L.lk_pyr_nlevels.argtypes = [C.c_void_p]
        L.lk_pyr_level_info.argtypes = [C.c_void_p, C.c_int] + [C.POINTER(C.c_int)] * 4
        L.lk_pyr_level_img.restype = C.c_void_p
        L.lk_pyr_level_img.argtypes = [C.c_void_p, C.c_int]
        L.lk_pyr_level_deriv.restype = C.c_void_p
        L.lk_pyr_level_deriv.argtypes = [C.c_void_p, C.c_int]
        L.lk_track.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                               C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_void_p]
        L.lk_set_sum_mode.argtypes = [C.c_int]
        L.lk_log_enable.argtypes = [C.c_void_p, C.c_longlong]
        L.lk_log_count.restype = C.c_longlong
        assert L.lk_log_record_size() == LK_EVENT.itemsize
        L.pyr_down_u8.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int]
        L.scharr_deriv.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int]
        L.fast_detect.restype = C.c_int
        L.fast_detect.argtypes = [C.c_void_p] + [C.c_int] * 5 + [C.c_void_p, C.c_void_p, C.c_int]
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def pyr_down(img):
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape
    out = np.zeros(((h + 1) // 2, (w + 1) // 2), np.uint8)
    lib().pyr_down_u8(_p(img), w, h, w, _p(out), out.shape[1])
    return out


def scharr(img):
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape
    out = np.zeros((h, w, 2), np.int16)
    lib().scharr_deriv(_p(img), w, h, w, _p(out), 2 * w)
    return out


class Pyramid:
    def __init__(self, img, win=21, max_level=3, with_deriv=True):
        img = np.ascontiguousarray(img, np.uint8)
        self._img = img
        h, w = img.shape
        self.h = lib().lk_pyr_build(_p(img), w, h, w, win, max_level, int(with_deriv))
        self.with_deriv = with_deriv

    def nlevels(self):
        return lib().lk_pyr_nlevels(self.h)

    def level(self, l):
        """(padded u8 image, pad) of level l (copy)."""
        w = C.c_int(); h = C.c_int(); pad = C.c_int(); step = C.c_int()
        lib().lk_pyr_level_info(self.h, l, C.byref(w), C.byref(h), C.byref(pad), C.byref(step))
        n = step.value * (h.value + 2 * pad.value)
        buf = (C.c_uint8 * n).from_address(lib().lk_pyr_level_img(self.h, l))
        return np.frombuffer(buf, np.uint8).reshape(h.value + 2 * pad.value, step.value).copy(), pad.value

    def close(self):
        if self.h:
            lib().lk_pyr_free(self.h)
            self.h = None

    def __del__(self):
        self.close()


def lk_track(prev, nxt, pts, win=21, max_level=3, max_count=30, epsilon=0.01, min_eig=1e-3,
             prev_pyr=None, next_pyr=None, return_iters=False, return_log=False):
    """One calcOpticalFlowPyrLK call (flags=0, err requested) on the C restatement.  return_log: also the event log
    (a LK_EVENT array in the order the oracle made the decisions: levels coarse to fine, points, iterations)."""
    pp = prev_pyr or Pyramid(prev, win, max_level, True)
    np_ = next_pyr or Pyramid(nxt, win, max_level, False)
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
    n = len(pts)
    out = np.zeros((n, 2), np.float32); st = np.zeros(n, np.uint8); err = np.zeros(n, np.float32)
    it = np.zeros(n, np.int32)
    log = np.zeros(0, LK_EVENT)

    def run():
        lib().lk_track(pp.h, np_.h, _p(pts), _p(out), _p(st), _p(err), n, win, max_count, epsilon, min_eig, _p(it))

    if n and return_log:
        cap = n * pp.nlevels() * 8
        while True:                     # the oracle counts the records it could not store: re-run with that size
            log = np.zeros(cap, LK_EVENT)
            lib().lk_log_enable(_p(log), cap)
            try:
                run()
                cnt = lib().lk_log_count()
            finally:
                lib().lk_log_enable(None, 0)
            if cnt <= cap:
                break
            cap = cnt
        log = log[:cnt]
    elif n:
        run()
    res = (out, st, err) + ((it,) if return_iters else ()) + ((log,) if return_log else ())
    return res


def fast_detect(img, threshold=20, nms=True, cap=None):
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape
    cap = cap or w * h
    xy = np.zeros((cap, 2), np.float32); resp = np.zeros(cap, np.float32)
    n = lib().fast_detect(_p(img), w, h, w, threshold, int(nms), _p(xy), _p(resp), cap)
    return xy[:n].copy(), resp[:n].copy()
