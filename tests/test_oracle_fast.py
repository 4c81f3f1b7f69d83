"""Pins the FAST restatement (oracle/fast_ref.c) list-exact against cv2 4.13.0's FastFeatureDetector (TYPE_9_16) on
images built to sit on FAST's edges, at thresholds 0..255 with and without non-max suppression.

The image set is defined here once, as module-level functions of the geometry, and tests/test_gpu_fast.py runs the
same images through the GPU detector:
  * uniform, low-contrast ([100, 140]) and binary (0 / 255) noise;
  * the dense 2x4 tile, which gives the most corners strict 3x3 non-max suppression allows;
  * a ring atlas: isolated patches whose 16 ring pixels hold arcs of 8, 9, 12 and 16 pixels at all 16 rotations,
    brighter and darker than the centre, at a contrast of exactly t and t+1 (both sides of `> v + t`), graded along the
    arc so the arc minimum moves through every arc position, or notched by one pixel at contrast t; plus saturated
    patches (0 inside 255 and the reverse) that score 254;
  * a tie atlas: small blobs of 1..9 pixels whose centres score equally (ties and plateaus under non-max suppression)
    or differ by one.
"""
import numpy as np
import pytest

THRESHOLDS = (0, 1, 7, 20, 100, 254, 255)

# the 16-pixel Bresenham ring of FAST-9/16, in cv2's order
RING_DX = (0, 1, 2, 3, 3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1)
RING_DY = (3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1, 0, 1, 2, 3)

TILE = np.array([[0, 0, 255, 0], [255, 0, 0, 0]], np.uint8)


def tile_to(pattern, h, w):
    """`pattern` repeated over an h x w frame (top-left aligned)."""
    ph, pw = pattern.shape
    return np.ascontiguousarray(np.tile(pattern, (-(-h // ph), -(-w // pw)))[:h, :w])


def uniform_noise(h, w, seed=1):
    return np.random.default_rng(seed).integers(0, 256, (h, w)).astype(np.uint8)


def low_contrast_noise(h, w, seed=2):
    return np.random.default_rng(seed).integers(100, 141, (h, w)).astype(np.uint8)


def binary_noise(h, w, seed=3):
    return (np.random.default_rng(seed).integers(0, 2, (h, w)) * 255).astype(np.uint8)


def dense_tile(h, w):
    return tile_to(TILE, h, w)


def nms_bound(h, w):
    """Most corners strict 3x3 non-max suppression can keep: one per 2x2 block of the (w-6) x (h-6) interior."""
    return -(-max(w - 6, 0) // 2) * -(-max(h - 6, 0) // 2)


ATLAS_CELL = 11
ATLAS_ARCS = (8, 9, 12, 16)
ATLAS_KINDS = ("t", "t+1", "graded", "notch")


def _ring_patches(t):
    """[(centre value, ring values[16], ring contrast > t mask[16])] of the ring atlas at threshold t."""
    v_lo = max(0, (254 - t) // 2)                     # v + (t+1) <= 255 whenever t <= 254
    out = []
    for L in ATLAS_ARCS:
        for rot in range(16):
            for kind in ATLAS_KINDS:
                c = np.zeros(16, np.int64)             # contrast of every ring pixel (0 off the arc)
                for j in range(L):
                    k = (rot + j) & 15
                    if kind == "t":
                        c[k] = t
                    elif kind == "t+1":
                        c[k] = t + 1
                    elif kind == "graded":              # unique arc minimum at arc position rot % L
                        c[k] = t + 1 + abs(j - rot % L)
                    else:                                # "notch": one pixel at t, at arc position rot % L
                        c[k] = t if j == rot % L else t + 1
                for sign in (1, -1):
                    v = v_lo if sign > 0 else 255 - v_lo
                    ring = np.clip(v + sign * c, 0, 255)
                    out.append((v, ring, sign * (ring - v) > t))
    out.append((0, np.full(16, 255), np.full(16, 255 > t)))       # saturated: score 254 below t = 255
    out.append((255, np.zeros(16, np.int64), np.full(16, 255 > t)))
    return out


def _has_arc9(mask):
    m = np.concatenate([mask, mask])
    run = 0
    for b in m:
        run = run + 1 if b else 0
        if run >= 9:
            return True
    return False


def ring_atlas_pattern(t):
    """(image, centres that are FAST corners at threshold t as an (n, 2) x, y array) of the ring atlas."""
    patches = _ring_patches(t)
    cols = 24
    rows = -(-len(patches) // cols)
    img = np.zeros((rows * ATLAS_CELL, cols * ATLAS_CELL), np.uint8)
    corners = []
    for i, (v, ring, mask) in enumerate(patches):
        y0, x0 = (i // cols) * ATLAS_CELL, (i % cols) * ATLAS_CELL
        img[y0:y0 + ATLAS_CELL, x0:x0 + ATLAS_CELL] = v
        cy, cx = y0 + ATLAS_CELL // 2, x0 + ATLAS_CELL // 2
        for k in range(16):
            img[cy + RING_DY[k], cx + RING_DX[k]] = ring[k]
        if _has_arc9(mask):
            corners.append((cx, cy))
    return img, np.array(corners, np.float32).reshape(-1, 2)


def ring_atlas(h, w, t):
    return tile_to(ring_atlas_pattern(t)[0], h, w)


TIE_CELL = 10
TIE_SHAPES = (((0, 0),), ((0, 0), (0, 1)), ((0, 0), (1, 0)), ((0, 0), (1, 1)), ((0, 0), (1, -1)),
              ((0, 0), (0, 1), (1, 0), (1, 1)), ((0, -1), (0, 0), (0, 1)), ((-1, 0), (0, 0), (1, 0)),
              tuple((dy, dx) for dy in (-1, 0, 1) for dx in (-1, 0, 1)), ((0, 0), (0, 1), (1, 0)))


TIE_COLOURS = ((255, 0), (0, 255), (200, 60), (60, 200), (130, 100))     # (background, blob)


def _tie_cells():
    return [(shape, bg, fg, step) for shape in TIE_SHAPES for bg, fg in TIE_COLOURS for step in (0, 1)]


def tie_cell_centre(i):
    """(x, y) of the blob origin of cell i of the tie atlas."""
    return (i % 10) * TIE_CELL + TIE_CELL // 2, (i // 10) * TIE_CELL + TIE_CELL // 2


def tie_atlas_pattern():
    """Blobs on a flat cell.  step 0: every blob pixel has the same value, so blob pixels that are corners tie;
    step 1: the first pixel is one level closer to the background, so it scores one less than the rest."""
    cells = _tie_cells()
    rows = -(-len(cells) // 10)
    img = np.zeros((rows * TIE_CELL, 10 * TIE_CELL), np.uint8)
    for i, (shape, bg, fg, step) in enumerate(cells):
        y0, x0 = (i // 10) * TIE_CELL, (i % 10) * TIE_CELL
        img[y0:y0 + TIE_CELL, x0:x0 + TIE_CELL] = bg
        cx, cy = tie_cell_centre(i)
        for j, (dy, dx) in enumerate(shape):
            img[cy + dy, cx + dx] = fg + (step * (1 if bg > fg else -1) if j == 0 else 0)
    return img


def tie_atlas(h, w):
    return tile_to(tie_atlas_pattern(), h, w)


def image_set(h, w, t):
    """name -> h x w image of every member of the set (the ring atlas depends on the threshold)."""
    return dict(uniform=uniform_noise(h, w), low_contrast=low_contrast_noise(h, w), binary=binary_noise(h, w),
                tile=dense_tile(h, w), ring_atlas=ring_atlas(h, w, t), ties=tie_atlas(h, w))


IMAGE_NAMES = ("uniform", "low_contrast", "binary", "tile", "ring_atlas", "ties")
SET_H, SET_W = 200, 300          # the geometry the parameter sweeps run at


def cv2_fast(img, threshold, nms):
    """cv2's FAST as the reference calls it: (xy (n, 2) f32 in keypoint order, response (n,) f32)."""
    cv2 = pytest.importorskip("cv2")
    kps = cv2.FastFeatureDetector_create(int(threshold), bool(nms)).detect(img)
    return (np.array([k.pt for k in kps], np.float32).reshape(-1, 2),
            np.array([k.response for k in kps], np.float32))


@pytest.mark.parametrize("nms", [1, 0])
@pytest.mark.parametrize("t", THRESHOLDS)
@pytest.mark.parametrize("name", IMAGE_NAMES)
def test_oracle_matches_cv2(built, name, t, nms):
    from oracle import cref
    img = image_set(SET_H, SET_W, t)[name]
    xy, resp = cref.fast_detect(img, threshold=t, nms=bool(nms))
    cxy, cresp = cv2_fast(img, t, nms)
    assert len(xy) == len(cxy)
    assert np.array_equal(xy, cxy)                     # coordinates and raster order
    assert np.array_equal(resp, cresp)
    if not nms:
        assert not resp.any()                          # cv2 scores nothing without non-max suppression


@pytest.mark.parametrize("t", THRESHOLDS)
def test_ring_atlas_centres(built, t):
    """The atlas is what it claims to be: without non-max suppression exactly the centres with >= 9 contiguous ring pixels
    beyond t are corners among the centres (t+1 arcs of 9..16 pixels yes, arcs of 8 and contrast-t arcs no)."""
    from oracle import cref
    img, expect = ring_atlas_pattern(t)
    xy, _ = cref.fast_detect(img, threshold=t, nms=False)
    centres = {(x, y) for x in range(ATLAS_CELL // 2, img.shape[1], ATLAS_CELL)
               for y in range(ATLAS_CELL // 2, img.shape[0], ATLAS_CELL)}
    got = {(int(x), int(y)) for x, y in xy} & centres
    assert got == {(int(x), int(y)) for x, y in expect}
    if t < 255:
        assert len(expect) > 100
    else:
        assert len(xy) == 0


def test_tie_atlas_has_ties(built):
    """The tie atlas holds what it claims: a pair of equal blob pixels are both corners, and non-max suppression keeps
    neither of them (equal scores are not strictly greater); with one of them a level closer to the background, the
    other one is kept."""
    from oracle import cref
    img = tie_atlas_pattern()
    off = {(int(x), int(y)) for x, y in cref.fast_detect(img, threshold=20, nms=False)[0]}
    on = {(int(x), int(y)) for x, y in cref.fast_detect(img, threshold=20, nms=True)[0]}
    cells = _tie_cells()
    for colours in TIE_COLOURS[:4]:
        i = cells.index((TIE_SHAPES[1], *colours, 0))                       # horizontal pair, equal
        cx, cy = tie_cell_centre(i)
        assert {(cx, cy), (cx + 1, cy)} <= off and not {(cx, cy), (cx + 1, cy)} & on
        i = cells.index((TIE_SHAPES[1], *colours, 1))                       # horizontal pair, first one level closer
        cx, cy = tie_cell_centre(i)
        assert (cx + 1, cy) in on and (cx, cy) not in on


@pytest.mark.parametrize("w,h,n", [(1241, 376, 114145), (1920, 1080, 513909)])
def test_dense_tile_exceeds_old_cap(built, w, h, n):
    """The tile is denser than w*h/8 corners; at 1920 x 1080 it reaches the non-max suppression bound exactly."""
    from oracle import cref
    img = dense_tile(h, w)
    xy, resp = cref.fast_detect(img)
    cxy, cresp = cv2_fast(img, 20, True)
    assert len(xy) == n and np.array_equal(xy, cxy) and np.array_equal(resp, cresp)
    assert n > max(w * h // 8, 65536) and n <= nms_bound(h, w)
    if (w, h) == (1920, 1080):
        assert n == nms_bound(h, w)


def test_threshold_zero_keeps_score_zero_corners(built):
    """At threshold 0 a corner whose best arc is one level beyond its centre scores 0; without non-max suppression it
    is still a corner (cv2: 23057 corners on this noise image), with it it can never be a strict maximum."""
    from oracle import cref
    img = uniform_noise(200, 300)
    xy, _ = cref.fast_detect(img, threshold=0, nms=False)
    cxy, _ = cv2_fast(img, 0, False)
    assert len(xy) == len(cxy) == 23057
