"""The training datasets' image steps after decoding (TEST INFRASTRUCTURE ONLY): cases and the generator of their golden.

`case(...)` builds a seeded synthetic decoded image, mask and camera: the image uniform uint8, the mask a disc of 1 with a
border of 100 and a patch of 13 (the values upstream's get_mask and the People-Snapshot masks carry) over 0, the camera a
pinhole with its centre off the pixel grid and the given distortion.  `cv2_steps(...)` runs upstream's host steps on it
with OpenCV (undistort of the float image and of the mask, INTER_AREA / INTER_NEAREST resize, background).

    python -m tools.item_images_case

writes, overwriting it, tests/golden/item_images.npz: small cases (every distortion kind, ratio 1 and 0.5, black and
white background) with OpenCV's outputs, so a machine without OpenCV checks nb_item_images and oracle/item_images.py
against them."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden", "item_images.npz")
# distortion kinds: a strong k1 that pulls the borders out of frame, tangential terms, the 8-coefficient rational model, none
DIST = {"k1": [0.6, 0.25, 0., 0., 0.05], "tangential": [-0.2, 0.05, 0.004, -0.003], "rational8": [-0.3, 0.1, 0.002,
        0.001, 0.01, 0.05, -0.02, 0.01], "zero": [0., 0., 0., 0., 0.]}
# (H0, W0, ratio, distortion, background: 0 none / 1 black / 2 white, seed)
GOLDEN_CASES = ((48, 64, 0.5, "k1", 1, 0), (40, 30, 1.0, "rational8", 2, 1), (36, 52, 0.5, "tangential", 0, 2),
                (30, 40, 1.0, "zero", 1, 3))


def case(H0, W0, dist, seed):
    """-> img_u8 (H0,W0,3), msk_u8 (H0,W0) uint8, K (3,3) float64, D (n,1) float64."""
    rng = np.random.RandomState(seed)
    img = rng.randint(0, 256, (H0, W0, 3)).astype(np.uint8)
    ys, xs = np.mgrid[:H0, :W0]
    r = np.hypot((ys - H0 * 0.5) / H0, (xs - W0 * 0.45) / W0)
    msk = np.zeros((H0, W0), np.uint8)
    msk[r < 0.3] = 1
    msk[(r >= 0.3) & (r < 0.34)] = 100
    msk[(r < 0.08)] = 13
    f = 1.1 * max(H0, W0)
    K = np.array([[f, 0., W0 * 0.5 + 0.37], [0., f * 1.01, H0 * 0.5 - 0.61], [0., 0., 1.]])
    D = np.array(DIST[dist], np.float64)[:, None]
    return img, msk, K, D


def cv2_steps(img_u8, msk_u8, K, D, ratio, bkgd):
    """Upstream's host steps (monocular_dataset.py:75-101) with OpenCV -> img (H,W,3) float32, msk (H,W) uint8."""
    import cv2
    img = cv2.undistort(img_u8.astype(np.float32) / 255., K, D)
    msk = cv2.undistort(msk_u8, K, D)
    H, W = int(img.shape[0] * ratio), int(img.shape[1] * ratio)
    img = cv2.resize(img, (W, H), interpolation=cv2.INTER_AREA)
    msk = cv2.resize(msk, (W, H), interpolation=cv2.INTER_NEAREST)
    if bkgd:
        img[msk == 0] = 0
        if bkgd == 2:
            img[msk == 0] = 1
    return img, msk


def load_golden():
    z = np.load(GOLDEN)
    out = []
    for c in range(len(GOLDEN_CASES)):
        out.append({k: z["c%d_%s" % (c, k)] for k in ("img_u8", "msk_u8", "K", "D", "ratio", "bkgd", "img", "msk")})
    return out


def main():
    import cv2
    arrays = {"cv2_version": np.frombuffer(cv2.__version__.encode(), np.uint8)}
    for c, (H0, W0, ratio, dist, bkgd, seed) in enumerate(GOLDEN_CASES):
        img_u8, msk_u8, K, D = case(H0, W0, dist, seed)
        img, msk = cv2_steps(img_u8, msk_u8, K, D, ratio, bkgd)
        for k, v in (("img_u8", img_u8), ("msk_u8", msk_u8), ("K", K), ("D", D), ("ratio", np.float64(ratio)),
                     ("bkgd", np.int64(bkgd)), ("img", img), ("msk", msk)):
            arrays["c%d_%s" % (c, k)] = v
    np.savez_compressed(GOLDEN, **arrays)
    print("wrote", GOLDEN)


if __name__ == "__main__":
    main()
