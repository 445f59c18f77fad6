"""The demo and mesh datasets' mask views after decoding (TEST INFRASTRUCTURE ONLY): the numpy restatement of the steps
nb_mask_views runs, seeded cases, OpenCV's steps, and the generator of their golden.

The restatement (`mask_view`) takes oracle/item_images.py's undistortion map and fixed-point remap and adds what the mask
views need beyond the training items' steps, as pinned by tests/test_mask_views_cpu.py against the cv2 the tests run with:
  - the binarisation (m != 0) of upstream's get_mask, before the undistort;
  - cv2.dilate(m, np.ones((5, 5), np.uint8)) with the default anchor, one iteration and the default border: each pixel
    becomes the maximum of the 5 x 5 window centred on it, pixels outside the image not taking part;
  - INTER_NEAREST at 2x: source pixel (2y, 2x).  Same size: a copy.

`case(...)` builds a seeded synthetic silhouette (two overlapping ellipses and a thin limb over 0, in one of three value
sets: {0, 1}, {0, 255} or arbitrary 0..255, as upstream's mask_cihp part labels are) and a pinhole camera with its centre
off the pixel grid and the given distortion.

    python -m tools.mask_views_case

writes, overwriting it, tests/golden/mask_views.npz: one small multi-view case per drop-in recipe (every view its own
camera) with OpenCV's outputs, so a machine without OpenCV checks nb_mask_views and the restatement against them."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.item_images import near_tie, reduction, remap, undistort_uv   # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "mask_views.npz")
# (binarise, dilate, resize by cfg.ratio) of each drop-in's masks
RECIPES = {"multi_view_demo": (True, 5, True), "multi_view_perform": (True, 5, True), "monocular_demo": (False, 0, True),
           "multi_view_mesh": (True, 5, False), "monocular_mesh": (False, 0, True)}
DIST = {"k1": [0.6, 0.25, 0., 0., 0.05], "d4": [-0.2, 0.05, 0.004, -0.003], "d5": [-0.25, 0.12, 0.001, -0.002, -0.03],
        "rational8": [-0.3, 0.1, 0.002, 0.001, 0.01, 0.05, -0.02, 0.01], "zero": [0., 0., 0., 0., 0.]}
VALUES = ("01", "0255", "any")
# golden cases: (recipe, H0, W0, ratio, views' distortions, value set, seed)
GOLDEN_CASES = (("multi_view_demo", 48, 64, 0.5, ("d5", "k1", "rational8"), "any", 0),
                ("multi_view_perform", 40, 52, 0.5, ("d5", "d4"), "01", 1),
                ("monocular_demo", 36, 30, 1.0, ("d4",), "any", 2),
                ("multi_view_mesh", 30, 44, 1.0, ("d5", "zero", "k1"), "0255", 3),
                ("monocular_mesh", 44, 40, 0.5, ("rational8",), "any", 4))


def dilate(m, size):
    """cv2.dilate(m, np.ones((size, size), np.uint8)) of a (H,W) uint8 array; size 0 is the identity."""
    if not size:
        return m
    r = size // 2
    H, W = m.shape
    p = np.zeros((H + 2 * r, W + 2 * r), np.uint8)      # 0 never wins a maximum of uint8 values
    p[r:r + H, r:r + W] = m
    out = np.zeros_like(m)
    for dy in range(size):
        for dx in range(size):
            np.maximum(out, p[dy:dy + H, dx:dx + W], out=out)
    return out


def mask_view(msk_u8, K, D, H, W, binarise, dilate_size):
    """One view's steps: msk_u8 (H0,W0) uint8 as decoded, the camera K, D at that size, the output size and the recipe.
    -> msk (H,W) uint8, ties (H,W) bool (an output pixel whose value reads a source pixel near a rounding tie)."""
    H0, W0 = msk_u8.shape
    k = reduction(H0, W0, H, W)
    src = (msk_u8 != 0).astype(np.uint8) if binarise else msk_u8
    U, V = undistort_uv(K, D, H0, W0)
    m = dilate(remap(src, U, V), dilate_size)
    tie = dilate((near_tie(U) | near_tie(V)).astype(np.uint8), dilate_size).astype(bool)
    return m[::k, ::k].copy(), tie[::k, ::k].copy()


def cv2_mask_view(msk_u8, K, D, H, W, binarise, dilate_size):
    """The same steps with OpenCV, as upstream's datasets run them on the host."""
    import cv2
    m = (msk_u8 != 0).astype(np.uint8) if binarise else msk_u8
    m = cv2.undistort(m, K, D)
    if dilate_size:
        m = cv2.dilate(m.copy(), np.ones((dilate_size, dilate_size), np.uint8))
    if m.shape != (H, W):
        m = cv2.resize(m, (W, H), interpolation=cv2.INTER_NEAREST)
    return m


def silhouette(H0, W0, values, seed):
    """A seeded (H0,W0) uint8 silhouette: 0 outside, inside {1}, {255} or part labels 1..255 (values '01', '0255',
    'any'; 'any' also scatters labels over the background, so an unbinarised view carries every kind of value)."""
    rng = np.random.RandomState(seed)
    ys, xs = np.mgrid[:H0, :W0].astype(np.float64)
    cy, cx = H0 * rng.uniform(0.4, 0.6), W0 * rng.uniform(0.4, 0.6)
    body = ((ys - cy) / (0.3 * H0)) ** 2 + ((xs - cx) / (0.18 * W0)) ** 2 < 1
    head = ((ys - cy + 0.38 * H0) / (0.1 * H0)) ** 2 + ((xs - cx) / (0.08 * W0)) ** 2 < 1
    limb = (np.abs(ys - cy - 0.6 * (xs - cx)) < 0.02 * H0 + 1) & (np.abs(xs - cx) < 0.4 * W0)
    inside = body | head | limb
    if values == "01":
        return inside.astype(np.uint8)
    if values == "0255":
        return inside.astype(np.uint8) * 255
    lab = rng.randint(1, 256, (H0, W0)).astype(np.uint8)
    m = np.where(inside, lab, 0).astype(np.uint8)
    spots = rng.rand(H0, W0) < 0.01
    m[spots] = lab[spots]
    return m


def camera(H0, W0, dist, seed):
    """A pinhole K (3,3) float64 with its centre off the pixel grid, and D (n,1) float64 of the named distortion."""
    rng = np.random.RandomState(1000 + seed)
    f = max(H0, W0) * rng.uniform(0.9, 1.3)
    K = np.array([[f, 0., W0 * 0.5 + rng.uniform(-3, 3)], [0., f * rng.uniform(0.98, 1.02), H0 * 0.5 + rng.uniform(-3, 3)],
                  [0., 0., 1.]])
    return K, np.array(DIST[dist], np.float64)[:, None]


def case(H0, W0, dists, values, seed):
    """-> msks_u8 (nv,H0,W0) uint8, Ks (nv,3,3) float64, Ds: nv (n,1) float64 arrays, one view per distortion."""
    msks = np.stack([silhouette(H0, W0, values, seed * 17 + v) for v in range(len(dists))])
    cams = [camera(H0, W0, d, seed * 17 + v) for v, d in enumerate(dists)]
    return msks, np.stack([K for K, _ in cams]), [D for _, D in cams]


def out_size(H0, W0, ratio):
    return int(H0 * ratio), int(W0 * ratio)


# ----------------------------------------------------------------------------- stand-ins for upstream's datasets
DROP_INS = {"multi_view_demo": "multi_view_demo_dataset", "multi_view_perform": "multi_view_perform_dataset",
            "monocular_demo": "monocular_demo_dataset", "multi_view_mesh": "multi_view_mesh_dataset",
            "monocular_mesh": "monocular_mesh_dataset"}
MONOCULAR = ("monocular_demo", "monocular_mesh")


def _prepare_input(*_):
    cb = np.array([[-0.5, -0.5, 1.5], [0.5, 0.5, 2.5]], np.float32)
    return (np.zeros((4, 3), np.int32), np.array([32, 32, 32], np.int32), cb, cb.copy(), np.zeros((1, 3)),
            np.zeros((1, 3), np.float32))


def stand_in(kind, H0, W0, nv, ratio, seed=0, values="01"):
    """A stand-in for upstream's Dataset of drop-in `kind` with the attributes the drop-in reads, over seeded decoded
    masks of H0 x W0 (two frames; `nv` views, 1 for the monocular sets) -> (Base class, imread, cfg keys).  Its host
    mask steps are upstream's recipe with OpenCV: the multi-view sets' get_mask binarises, undistorts with the view's K
    (the demo sets store it scaled by cfg.ratio, as upstream's __init__ does) and dilates by 5 x 5."""
    import cv2
    nv = 1 if kind in MONOCULAR else nv
    dists = ("rational8",) if kind in MONOCULAR else ("d5", "k1", "zero")    # upstream stacks the views' D
    files, Ks, Ds = {}, [], []
    for v in range(nv):
        K, D = camera(H0, W0, dists[v % len(dists)], seed * 31 + v)
        Ks.append(K)
        Ds.append(D)
        for f in range(2):
            m = silhouette(H0, W0, values, seed * 31 + 7 * v + f)
            files["/zju/mask_cihp/%02d/%06d.png" % (v, f)] = m
            files["/snap/mask/%d.png" % f] = m
    imread = lambda p: files[p].copy()
    cfg = dict(H=H0, W=W0, ratio=ratio, ith_frame=1, begin_ith_frame=0, num_train_frame=2)
    scaled = kind in ("multi_view_demo", "multi_view_perform")

    class Base:
        def __init__(self):
            if kind in MONOCULAR:
                self.data_root, self.begin_ith_frame = "/snap", 0
                # snapshot_data_utils.get_camera: float64 K, D; the demo drop-in casts K to float32 itself
                self.cam = {"K": Ks[0], "D": Ds[0].ravel(), "R": np.eye(3), "T": np.array([0., 0., 2.])}
                self.params = {"pose": np.zeros((2, 72), np.float32), "trans": np.zeros((2, 3), np.float32)}
                return
            self.data_root = "/zju"
            self.ims = np.array([["%02d/%06d.jpg" % (v, f) for v in range(nv)] for f in range(2)])
            Kf = np.stack(Ks).astype(np.float32)
            if scaled:
                Kf[:, :2] = Kf[:, :2] * ratio
            self.Ks, self.Ds = Kf, np.stack(Ds).astype(np.float32)
            self.K = self.Ks[0]
            self.RT = np.tile(np.eye(4, dtype=np.float32)[:3], (nv, 1, 1))
            self.Rs, self.Ts = np.tile(np.eye(3, dtype=np.float32), (nv, 1, 1)), np.zeros((nv, 3, 1), np.float32)
            self.render_w2c = [np.eye(4)[:3] for _ in range(3)]

        def _host_mask(self, i, v):
            m = (imread(os.path.join(self.data_root, "mask_cihp", self.ims[i][v])[:-4] + ".png") != 0).astype(np.uint8)
            K = self.Ks[v].copy()
            if scaled:
                K[:2] = K[:2] / ratio
            m = cv2.undistort(m, K, self.Ds[v])
            return cv2.dilate(m.copy(), np.ones((5, 5), np.uint8))

        def get_mask(self, i, v=None):
            return self._host_mask(i, v) if v is not None else [self._host_mask(i, u) for u in range(len(self.ims[i]))]

        def prepare_input(self, *a):
            return _prepare_input(*a)
    return Base, imread, cfg


def make_item(kind, Base, imread, index):
    """Item `index` of drop-in `kind` over the stand-in (OpenCV as the drop-in's cv2)."""
    import importlib
    mod = importlib.import_module("neuralbody_b200.lib.datasets.light_stage." + DROP_INS[kind])
    if kind == "multi_view_mesh":
        import cv2
        return mod.make_dataset_class(Base, rodrigues=cv2.Rodrigues, imread=imread)()[index]
    return mod.make_dataset_class(Base, imread=imread)()[index]


def with_cfg(new):
    """Set the active config's keys `new` -> a function restoring them."""
    from neuralbody_b200.lib.config import get_active_cfg
    cfg = get_active_cfg()
    old = {k: cfg[k] for k in new if k in cfg}
    dict.update(cfg, new)

    def restore():
        for k in new:
            dict.pop(cfg, k, None)
        dict.update(cfg, old)
    return restore


def item_pair(kind, H0, W0, nv, ratio, seed=0, values="01", index=1):
    """The 'host' and 'device' items of drop-in `kind` built from the same decoded masks."""
    Base, imread, cfg = stand_in(kind, H0, W0, nv, ratio, seed, values)
    out = []
    for steps in ("host", "device"):
        restore = with_cfg(dict(cfg, dataset_image_steps=steps))
        try:
            out.append(make_item(kind, Base, imread, index))
        finally:
            restore()
    return tuple(out)


def restate_item(item):
    """The restatement of a 'device' item's mask steps from its msks_u8 and meta -> (msks (nv,H,W), ties (nv,H,W))."""
    m = item["meta"]
    H, W = (int(v) for v in m["mask_size"])
    got = [mask_view(u, c[:9].reshape(3, 3), c[9:9 + int(m["mask_n_dist"])], H, W, bool(m["mask_binarise"]),
                     int(m["mask_dilate"])) for u, c in zip(item["msks_u8"], m["mask_cams"])]
    return np.stack([g for g, _ in got]), np.stack([t for _, t in got])


def load_golden():
    z = np.load(GOLDEN)
    out = []
    for c, (recipe, _, _, ratio, dists, _, _) in enumerate(GOLDEN_CASES):
        g = {k: z["c%d_%s" % (c, k)] for k in ("msks_u8", "Ks", "msks")}
        g["Ds"] = [z["c%d_D%d" % (c, v)] for v in range(len(dists))]
        g["recipe"], g["ratio"] = recipe, ratio
        out.append(g)
    return out


def main():
    import cv2
    arrays = {"cv2_version": np.frombuffer(cv2.__version__.encode(), np.uint8)}
    for c, (recipe, H0, W0, ratio, dists, values, seed) in enumerate(GOLDEN_CASES):
        binarise, dil, _ = RECIPES[recipe]
        msks_u8, Ks, Ds = case(H0, W0, dists, values, seed)
        H, W = out_size(H0, W0, ratio)
        arrays["c%d_msks_u8" % c], arrays["c%d_Ks" % c] = msks_u8, Ks
        for v, D in enumerate(Ds):
            arrays["c%d_D%d" % (c, v)] = D
        arrays["c%d_msks" % c] = np.stack([cv2_mask_view(m, K, D, H, W, binarise, dil) for m, K, D in zip(msks_u8, Ks, Ds)])
    np.savez_compressed(GOLDEN, **arrays)
    print("wrote", GOLDEN)


if __name__ == "__main__":
    main()
