"""numpy restatement of the training datasets' image steps after decoding, as nb_item_images runs them on the device:
cv2.undistort of the float image and of the uint8 mask, the INTER_AREA / INTER_NEAREST resize by cfg.ratio (a copy, or an
exact 2x reduction), the background fill and the sampler's class map (multi_view_dataset.py:121-145,
monocular_dataset.py:74-103 upstream; neuralbody_b200.lib.datasets.train_item for the class rules).

What OpenCV does, as pinned by tests/test_item_images_cpu.py against the cv2 the tests run with:
  - cv::undistort builds its map in stripes of max(1, 4096 // W) rows.  Per stripe it inverts the new camera matrix (the
    camera matrix with Ar(1,2) = cy - y0) by the 3x3 adjugate over the determinant (cv::invert's DECOMP_LU for n = 3), and
    initUndistortRectifyMap then walks each row from (i*ir[1] + ir[2], i*ir[4] + ir[5], i*ir[7] + ir[8]), adding ir[0],
    ir[3], ir[6] once per column: the map of a pixel depends on the sequence of sums before it in its row.
  - u, v are scaled by 32 (INTER_TAB_SIZE) and rounded to nearest-even into int32 (a NaN or an out-of-range value becomes
    INT_MIN, as SSE2's cvtsd2si); the integer part is (iu >> 5) saturated to int16, the fraction iu & 31.
  - remap, float32: sum = S00 w00 + S01 w01 + S10 w10 + S11 w11 in float32, left to right, with the table's float weights
    (1 - f, f) products, out-of-image neighbours 0 (BORDER_CONSTANT).  uint8: the same with the weights * 32768 as integers
    and (sum + 2^14) >> 15.
  - INTER_AREA at exactly 2x (resizeAreaFast, three channels): ((S00 + S01) + S10) + S11, then * 0.25f.  INTER_NEAREST at
    2x: source pixel (2y, 2x).  Same size: a copy.

A pixel whose u * 32 or v * 32 lies within TIE_EPS of a rounding tie (a half-integer) is flagged: there a restatement one
ulp away from OpenCV's arithmetic could round the other way."""
import numpy as np

NONE, H36M, SNAPSHOT = 0, 1, 2           # NB_ITEM_CLASS_*
BKGD_NONE, BKGD_BLACK, BKGD_WHITE = 0, 1, 2   # NB_ITEM_BKGD_*
BODY, FACE, BOUND = 1, 2, 4              # NB_TRAIN_CLASS_*
TIE_EPS = 1e-6                           # in units of 1/32 px
INT_MIN = -(1 << 31)


def dist_coeffs(D):
    """D with 4, 5 or 8 coefficients -> the 8 (k1, k2, p1, p2, k3, k4, k5, k6) OpenCV reads, zero-padded, float64."""
    d = np.asarray(D, dtype=np.float64).ravel()
    if d.size not in (4, 5, 8):
        raise ValueError("the distortion model must have 4, 5 or 8 coefficients (got %d)" % d.size)
    out = np.zeros(8)
    out[:d.size] = d
    return out


def inv3(m):
    """cv::invert(DECOMP_LU) of a 3x3 float64 matrix: the adjugate times 1 / det3, in OpenCV's order."""
    m = np.asarray(m, dtype=np.float64)
    det = (m[0, 0] * (m[1, 1] * m[2, 2] - m[1, 2] * m[2, 1]) - m[0, 1] * (m[1, 0] * m[2, 2] - m[1, 2] * m[2, 0])) + \
        m[0, 2] * (m[1, 0] * m[2, 1] - m[1, 1] * m[2, 0])
    d = 1. / det
    return np.array([(m[1, 1] * m[2, 2] - m[1, 2] * m[2, 1]) * d, (m[0, 2] * m[2, 1] - m[0, 1] * m[2, 2]) * d,
                     (m[0, 1] * m[1, 2] - m[0, 2] * m[1, 1]) * d, (m[1, 2] * m[2, 0] - m[1, 0] * m[2, 2]) * d,
                     (m[0, 0] * m[2, 2] - m[0, 2] * m[2, 0]) * d, (m[0, 2] * m[1, 0] - m[0, 0] * m[1, 2]) * d,
                     (m[1, 0] * m[2, 1] - m[1, 1] * m[2, 0]) * d, (m[0, 1] * m[2, 0] - m[0, 0] * m[2, 1]) * d,
                     (m[0, 0] * m[1, 1] - m[0, 1] * m[1, 0]) * d])


def undistort_uv(K, D, H, W):
    """The source position (u, v) float64 (H,W) cv2.undistort(src, K, D) samples for each destination pixel."""
    A = np.asarray(K, dtype=np.float64).reshape(3, 3)
    k1, k2, p1, p2, k3, k4, k5, k6 = dist_coeffs(D)
    fx, fy, u0, v0 = A[0, 0], A[1, 1], A[0, 2], A[1, 2]
    stripe = min(max(1, 4096 // W), H)
    ir = np.empty((H, 9))          # each row's stripe's inverse
    for y0 in range(0, H, stripe):
        Ar = A.copy()
        Ar[1, 2] = v0 - y0
        ir[y0:y0 + stripe] = inv3(Ar)
    i = (np.arange(H) % stripe).astype(np.float64)
    x_, y_, w_ = i * ir[:, 1] + ir[:, 2], i * ir[:, 4] + ir[:, 5], i * ir[:, 7] + ir[:, 8]
    X, Y, Wt = np.empty((W, H)), np.empty((W, H)), np.empty((W, H))
    for j in range(W):
        X[j], Y[j], Wt[j] = x_, y_, w_
        x_, y_, w_ = x_ + ir[:, 0], y_ + ir[:, 3], w_ + ir[:, 6]
    w = 1. / Wt.T
    x, y = X.T * w, Y.T * w
    x2, y2 = x * x, y * y
    r2 = x2 + y2
    _2xy = 2 * x * y
    with np.errstate(all="ignore"):
        kr = (1 + ((k3 * r2 + k2) * r2 + k1) * r2) / (1 + ((k6 * r2 + k5) * r2 + k4) * r2)
        U = fx * (x * kr + p1 * _2xy + p2 * (r2 + 2 * x2)) + u0
        V = fy * (y * kr + p1 * (r2 + 2 * y2) + p2 * _2xy) + v0
    return U, V


def fixed_point(c):
    """saturate_cast<int>(c * 32) as SSE2 rounds it, then (saturate_cast<short>(i >> 5), i & 31), int64 arrays."""
    with np.errstate(invalid="ignore"):
        r = np.rint(c * 32.)
        bad = ~((r >= INT_MIN) & (r <= (1 << 31) - 1))
    i = np.where(bad, INT_MIN, r).astype(np.int64)
    return np.clip(i >> 5, -32768, 32767), i & 31


def near_tie(c, eps=TIE_EPS):
    """Where c * 32 lies within eps of a half-integer."""
    with np.errstate(invalid="ignore"):
        t = c * 32.
        return np.abs(t - np.floor(t) - 0.5) < eps


def remap(src, U, V):
    """cv2.remap(src, map1, map2, INTER_LINEAR, BORDER_CONSTANT 0) with the CV_16SC2 / CV_16UC1 maps of (U, V); src float32
    (H,W,C) or uint8 (H,W)."""
    H, W = src.shape[:2]
    sx, fx = fixed_point(U)
    sy, fy = fixed_point(V)
    f32 = src.dtype == np.float32
    a, b = fx.astype(np.float32) * np.float32(1 / 32), fy.astype(np.float32) * np.float32(1 / 32)
    wts = [(np.float32(1) - b) * (np.float32(1) - a), (np.float32(1) - b) * a, b * (np.float32(1) - a), b * a]
    out = None
    for (dy, dx), w in zip(((0, 0), (0, 1), (1, 0), (1, 1)), wts):
        yy, xx = sy + dy, sx + dx
        ok = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
        s = src[np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)]
        if f32:
            s = np.where(ok[..., None], s, np.float32(0)) * w[..., None]
            out = s if out is None else out + s
        else:
            s = np.where(ok, s, 0).astype(np.int64) * (w * np.float32(32768)).astype(np.int64)
            out = s if out is None else out + s
    return out.astype(np.float32) if f32 else np.clip((out + (1 << 14)) >> 15, 0, 255).astype(np.uint8)


def reduction(H0, W0, H, W):
    """1 for a copy, 2 for an exact 2x reduction; ValueError for any other geometry."""
    if (H, W) == (H0, W0):
        return 1
    if (2 * H, 2 * W) == (H0, W0):
        return 2
    raise ValueError("the image steps resize %dx%d to %dx%d: only a copy or an exact 2x reduction is implemented"
                     % (H0, W0, H, W))


def class_map(rule, msk, bound):
    """train_item.class_map_h36m / class_map_snapshot as bits; None for NONE."""
    if rule == NONE:
        return None
    m = (msk * bound).astype(np.uint8)
    if rule == H36M:
        b = (bound == 1) & (m != 100)
        return ((m == 1) * BODY | (m == 13) * FACE | b * BOUND).astype(np.uint8)
    return ((m != 0) * BODY | (m == 13) * FACE | (bound == 1) * BOUND).astype(np.uint8)


def item_images(img_u8, msk_u8, K, D, H, W, bkgd=BKGD_NONE, rule=NONE, bound=None):
    """One item's steps: img_u8 (H0,W0,3), msk_u8 (H0,W0) uint8, the camera K, D at the source size, the output size.
    -> img (H,W,3) float32, msk (H,W) uint8, class map (H,W) uint8 or None, ties (H,W) bool (an output pixel one of whose
    source pixels lies near a rounding tie)."""
    H0, W0 = msk_u8.shape
    k = reduction(H0, W0, H, W)
    U, V = undistort_uv(K, D, H0, W0)
    img = remap(img_u8.astype(np.float32) / np.float32(255.), U, V)
    msk = remap(msk_u8, U, V)
    tie = near_tie(U) | near_tie(V)
    if k == 2:
        img = (((img[0::2, 0::2] + img[0::2, 1::2]) + img[1::2, 0::2]) + img[1::2, 1::2]) * np.float32(0.25)
        msk = msk[0::2, 0::2]
        tie = tie[0::2, 0::2] | tie[0::2, 1::2] | tie[1::2, 0::2] | tie[1::2, 1::2]
    if bkgd != BKGD_NONE:
        img[msk == 0] = 1 if bkgd == BKGD_WHITE else 0
    return img, msk, class_map(rule, msk, bound), tie
