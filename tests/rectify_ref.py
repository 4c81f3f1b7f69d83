"""A restatement of cv2.remap(INTER_LINEAR, BORDER_CONSTANT 0) on 8-bit images, in numpy, in cv2's fixed-point
arithmetic.  The tests hold it to cv2 bit for bit, and the library's kernel to it."""
import numpy as np

INTER_BITS = 5
INTER_TAB = 1 << INTER_BITS


def _round_int32(v):
    """cvRound of a float32 (round half to even); out of the int32 range or NaN: INT_MIN, as x86's cvtss2si gives."""
    v = np.asarray(v, np.float32)
    out = np.full(v.shape, np.iinfo(np.int32).min, np.int64)
    ok = np.isfinite(v) & (np.abs(v.astype(np.float64)) < 2.0 ** 31)
    out[ok] = np.rint(v[ok].astype(np.float64)).astype(np.int64)
    return out


def fixed_maps(map_x, map_y):
    """The fixed-point form cv2.remap makes of float maps: (sx, sy) = the integer part, saturated to int16, and
    a = the 5-bit fractions, fy * 32 + fx (what cv2.convertMaps(CV_16SC2) stores)."""
    X = _round_int32(np.asarray(map_x, np.float32) * np.float32(INTER_TAB))
    Y = _round_int32(np.asarray(map_y, np.float32) * np.float32(INTER_TAB))
    sx = np.clip(X >> INTER_BITS, -32768, 32767).astype(np.int16)
    sy = np.clip(Y >> INTER_BITS, -32768, 32767).astype(np.int16)
    a = ((Y & (INTER_TAB - 1)) * INTER_TAB + (X & (INTER_TAB - 1))).astype(np.uint16)
    return sx, sy, a


def remap_fixed(src, sx, sy, a):
    """cv2.remap(INTER_LINEAR, BORDER_CONSTANT 0) of an 8-bit gray image through fixed maps: 15-bit weights
    ((32 - fx) (32 - fy), fx (32 - fy), (32 - fx) fy, fx fy) * 32 that sum to 2^15, taps outside the image read 0,
    (sum + 2^14) >> 15."""
    src = np.asarray(src, np.uint8)
    h, w = src.shape
    sx = sx.astype(np.int64)
    sy = sy.astype(np.int64)
    fx = (a & 31).astype(np.int64)
    fy = (a >> 5).astype(np.int64)

    def tap(x, y):
        ok = (x >= 0) & (x < w) & (y >= 0) & (y < h)
        return np.where(ok, src[np.clip(y, 0, h - 1), np.clip(x, 0, w - 1)].astype(np.int64), 0)

    s = (tap(sx, sy) * ((32 - fx) * (32 - fy)) + tap(sx + 1, sy) * (fx * (32 - fy))
         + tap(sx, sy + 1) * ((32 - fx) * fy) + tap(sx + 1, sy + 1) * (fx * fy)) * 32
    return ((s + (1 << 14)) >> 15).astype(np.uint8)


def remap(src, map_x, map_y):
    return remap_fixed(src, *fixed_maps(map_x, map_y))


def gray_of(bgr):
    """cv2.cvtColor(BGR2GRAY)'s fixed point."""
    b, g, r = (bgr[..., k].astype(np.int64) for k in range(3))
    return ((b * 3735 + g * 19235 + r * 9798 + (1 << 14)) >> 15).astype(np.uint8)
