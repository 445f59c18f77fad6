"""The training datasets' image steps after decoding without a GPU: the numpy restatement (oracle/item_images.py) against
OpenCV, nb_item_images' argument validation, and the drop-ins' `dataset_image_steps` item kinds."""
import ctypes as C

import numpy as np
import pytest

from oracle import item_images as O
from tools import item_images_case as IC
from neuralbody_b200.lib.datasets import train_item


# ----------------------------------------------------------------------------- the restatement against OpenCV
GEOMETRIES = [(1024, 1024, 0.5), (1080, 1080, 1.0), (1080, 1080, 0.5), (1000, 1002, 1.0)]


@pytest.mark.parametrize("dist", sorted(IC.DIST))
@pytest.mark.parametrize("geom", GEOMETRIES, ids=["%dx%d_r%g" % g for g in GEOMETRIES])
def test_restatement_equals_cv2_outside_flagged_ties(geom, dist):
    """cv2.undistort + cv2.resize of the float image and of the mask equal the restatement at every pixel that is not
    flagged as lying within TIE_EPS of a 1/32 px rounding tie."""
    cv2 = pytest.importorskip("cv2")
    H0, W0, ratio = geom
    img_u8, msk_u8, K, D = IC.case(H0, W0, dist, seed=H0 + W0)
    want_img, want_msk = IC.cv2_steps(img_u8, msk_u8, K, D, ratio, bkgd=0)
    H, W = int(H0 * ratio), int(W0 * ratio)
    img, msk, _, tie = O.item_images(img_u8, msk_u8, K, D, H, W)
    bad_img = (img.view(np.uint32) != want_img.view(np.uint32)).any(-1)
    bad_msk = msk != want_msk
    print("%s %s: %d flagged pixels, %d of them differ" % (geom, dist, tie.sum(), (bad_img | bad_msk).sum()))
    assert not (bad_img & ~tie).any() and not (bad_msk & ~tie).any()
    assert tie.sum() <= 64
    if dist == "k1":
        U, V = O.undistort_uv(K, D, H0, W0)              # the corners sample outside the source: the borders go black
        assert U[0, 0] < -1 and V[0, 0] < -1 and U[-1, -1] > W0 and V[-1, -1] > H0
    assert cv2.__version__


def test_restatement_map_is_opencvs_map():
    """The (u, v) positions rounded to 1/32 px equal initUndistortRectifyMap's CV_16SC2 map, stripe by stripe, as
    cv::undistort builds it."""
    cv2 = pytest.importorskip("cv2")
    H0, W0 = 300, 1002
    _, _, K, D = IC.case(H0, W0, "rational8", 0)
    U, V = O.undistort_uv(K, D, H0, W0)
    stripe = max(1, 4096 // W0)
    for y0 in range(0, H0, stripe):
        n = min(stripe, H0 - y0)
        Ar = K.copy()
        Ar[1, 2] -= y0
        m1, m2 = cv2.initUndistortRectifyMap(K, D, np.eye(3), Ar, (W0, n), cv2.CV_16SC2)
        ix, fx = O.fixed_point(U[y0:y0 + n])
        iy, fy = O.fixed_point(V[y0:y0 + n])
        tie = O.near_tie(U[y0:y0 + n]) | O.near_tie(V[y0:y0 + n])
        ok = (m1[..., 0] == ix) & (m1[..., 1] == iy) & (m2.astype(np.int64) == fy * 32 + fx)
        assert (ok | tie).all(), y0


def test_restatement_saturates_as_opencv():
    """Far out-of-frame positions: the int32 conversion overflows to INT_MIN and the int16 map entry saturates, as in
    OpenCV; the image and mask still match."""
    pytest.importorskip("cv2")
    for k1 in (1e4, 1e9):
        img_u8, msk_u8, K, _ = IC.case(60, 40, "zero", 5)
        D = np.array([[k1], [0.], [0.], [0.]])
        want_img, want_msk = IC.cv2_steps(img_u8, msk_u8, K, D, 1.0, 0)
        img, msk, _, tie = O.item_images(img_u8, msk_u8, K, D, 60, 40)
        assert np.array_equal(img[~tie], want_img[~tie]) and np.array_equal(msk[~tie], want_msk[~tie])


def test_goldens_are_cv2s_and_the_restatements():
    """The small goldens the GPU tests read hold OpenCV's outputs, which the restatement reproduces."""
    for c, g in enumerate(IC.load_golden()):
        H0, W0 = g["msk_u8"].shape
        H, W = int(H0 * g["ratio"]), int(W0 * g["ratio"])
        img, msk, _, tie = O.item_images(g["img_u8"], g["msk_u8"], g["K"], g["D"], H, W, int(g["bkgd"]))
        assert np.array_equal(img[~tie], g["img"][~tie]) and np.array_equal(msk[~tie], g["msk"][~tie]), c
        try:
            import cv2  # noqa: F401
        except ImportError:
            continue
        want_img, want_msk = IC.cv2_steps(g["img_u8"], g["msk_u8"], g["K"], g["D"], float(g["ratio"]), int(g["bkgd"]))
        assert np.array_equal(want_img, g["img"]) and np.array_equal(want_msk, g["msk"]), c


def test_class_rules_are_train_items():
    rng = np.random.RandomState(0)
    msk = rng.choice(np.array([0, 1, 13, 100, 7], np.uint8), (20, 30))
    bound = (rng.rand(20, 30) < 0.7).astype(np.uint8)
    assert np.array_equal(O.class_map(O.H36M, msk, bound), train_item.class_map_h36m(msk, bound))
    assert np.array_equal(O.class_map(O.SNAPSHOT, msk, bound), train_item.class_map_snapshot(msk, bound))


def test_unsupported_geometry_and_models_raise():
    with pytest.raises(ValueError):
        O.reduction(101, 100, 50, 50)
    with pytest.raises(ValueError):
        O.dist_coeffs(np.zeros(6))
    from neuralbody_b200 import images
    with pytest.raises(ValueError):
        images.reduction(1000, 1000, 300, 300)
    for n in (3, 6, 12, 14):
        with pytest.raises(ValueError):
            images.item_camera(np.eye(3), np.zeros((n, 1)))
    n, cam = images.item_camera(np.eye(3, dtype=np.float32), np.array([[0.1, 0.2, 0.3, 0.4, 0.5]], np.float32))
    assert n == 5 and cam.dtype == np.float64 and cam[9:14].tolist() == [float(np.float32(v)) for v in (.1, .2, .3, .4, .5)]


# ----------------------------------------------------------------------------- C ABI validation
def _args(**kw):
    from neuralbody_b200 import capi
    a = capi.nb_item_images_args()
    a.B, a.H0, a.W0, a.H, a.W, a.n_dist = 1, 8, 6, 4, 3, 5
    a.bkgd, a.class_rule = capi.NB_ITEM_BKGD_BLACK, capi.NB_ITEM_CLASS_NONE
    a.img_u8 = a.msk_u8 = a.cams = a.img = a.msk = 256        # never dereferenced: validation fails before any launch
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def test_bad_arguments_are_rejected_before_any_launch():
    from neuralbody_b200 import capi
    L = capi.load()
    assert L.nb_item_images(None, None) == -1
    for field in ("img_u8", "msk_u8", "cams", "img", "msk"):
        assert L.nb_item_images(C.byref(_args(**{field: None})), None) == -1, field
        assert b"null" in L.nb_last_error()
    for kw in ({"B": 0}, {"H0": 0}, {"W0": 0}, {"W0": capi.NB_ITEM_MAX_W + 2, "W": capi.NB_ITEM_MAX_W // 2 + 1},
               {"B": 70000}):
        assert L.nb_item_images(C.byref(_args(**kw)), None) == -1, kw
        assert b"B in" in L.nb_last_error()
    for H, W in ((3, 3), (4, 4), (5, 3), (8, 5), (0, 0)):
        assert L.nb_item_images(C.byref(_args(H=H, W=W)), None) == -1 and b"half" in L.nb_last_error()
    for n in (0, 3, 6, 12, 14):
        assert L.nb_item_images(C.byref(_args(n_dist=n)), None) == -1 and b"n_dist" in L.nb_last_error()
    for b in (-1, 3):
        assert L.nb_item_images(C.byref(_args(bkgd=b)), None) == -1 and b"bkgd" in L.nb_last_error()
    for r in (-1, 3):
        assert L.nb_item_images(C.byref(_args(class_rule=r)), None) == -1 and b"class_rule" in L.nb_last_error()
    for kw in ({"class_rule": capi.NB_ITEM_CLASS_H36M}, {"class_rule": capi.NB_ITEM_CLASS_SNAPSHOT, "bound": 256},
               {"bound": 256, "class_map": 256}, {"class_map": 256}):
        assert L.nb_item_images(C.byref(_args(**kw)), None) == -1 and b"bound and class_map" in L.nb_last_error(), kw


# ----------------------------------------------------------------------------- the drop-ins' item kinds
class _Cv2Stub:
    INTER_AREA, INTER_NEAREST = 3, 0

    def __init__(self):
        self.calls = []

    def resize(self, a, size, interpolation=None):
        self.calls.append("resize")
        W, H = size
        return a[np.arange(H) * a.shape[0] // H][:, np.arange(W) * a.shape[1] // W].copy()

    def undistort(self, a, K, D):
        self.calls.append("undistort")
        return a.copy()

    def Rodrigues(self, r):
        return (np.eye(3), None)


def _prepare_input(i):
    cb = np.array([[-0.5, -0.5, 1.5], [0.5, 0.5, 2.5]], np.float32)
    return (np.zeros((4, 3), np.int32), np.array([32, 32, 32], np.int32), cb, cb.copy(), np.zeros((1, 3)),
            np.zeros((1, 3), np.float32))


def _mv_base(split, msk, K, D):
    class Base:
        def __init__(self):
            self.data_root, self.human, self.split, self.nrays = "/data", "CoreView_377", split, 500
            self.ims, self.cam_inds = np.array(["Camera_B1/000003.jpg"]), np.array([0])
            self.cams = {"K": [K], "D": [D], "R": [np.eye(3)], "T": [np.array([[0.], [0.], [2000.]])]}

        def get_mask(self, index):
            return msk.copy()

        def prepare_input(self, i):
            return _prepare_input(i)
    return Base


def _mono_base(split, K, D):
    class Base:
        def __init__(self):
            self.data_root, self.split, self.nrays = "/snap", split, 400
            self.cam = {"K": K, "D": D, "R": np.eye(3), "T": np.array([0., 0., 2.])}
            self.params = {"pose": np.zeros((4, 72), np.float32), "trans": np.zeros((4, 3), np.float32)}

        def prepare_input(self, i):
            return _prepare_input(i)
    return Base


def _with_cfg(new):
    from neuralbody_b200.lib.config import get_active_cfg
    cfg = get_active_cfg()
    old = {k: cfg[k] for k in new if k in cfg}
    dict.update(cfg, new)

    def restore():
        for k in new:
            dict.pop(cfg, k, None)
        dict.update(cfg, old)
    return restore


@pytest.mark.parametrize("kind", ["mv", "mono"])
@pytest.mark.parametrize("split", ["train", "test"])
def test_dropin_device_items(kind, split):
    """With dataset_image_steps 'device' the drop-ins stop after decoding: no cv2 image step runs, and the item carries
    the decoded image and mask, the camera, upstream's bound mask (split 'train') and the steps under 'meta', with the
    host item's camera and every other key.  With 'host' (and without the key) the item is the host item."""
    from neuralbody_b200.lib.datasets.light_stage import multi_view_dataset as mv, monocular_dataset as mono
    rng = np.random.RandomState(1)
    img_u8 = rng.randint(0, 256, (16, 12, 3)).astype(np.uint8)
    msk = np.zeros((16, 12), np.uint8)
    msk[4:12, 3:9] = 1
    K = np.array([[20., 0, 6], [0, 20, 8], [0, 0, 1]])
    D = np.array([[-0.1], [0.01], [0.], [0.], [0.]])
    bound = np.zeros((8, 6), np.uint8)
    bound[1:7, 1:5] = 1
    b2d = lambda cb, Kb, pose, H, W: bound.copy()
    if kind == "mv":
        make = lambda cv: mv.make_dataset_class(_mv_base(split, msk, K, D), cv2=cv, imread=lambda p: img_u8.copy(),
                                                bound_2d_mask=b2d)
    else:
        files = {"/snap/image/0.jpg": img_u8, "/snap/mask/0.png": msk}
        make = lambda cv: mono.make_dataset_class(_mono_base(split, K.astype(np.float32), D.ravel().astype(np.float32)),
                                                  cv2=cv, imread=lambda p: files[p].copy(), bound_2d_mask=b2d)
    base = dict(H=16, W=12, ratio=0.5, mask_bkgd=True, white_bkgd=True, body_sample_ratio=0.5, face_sample_ratio=0.0,
                begin_ith_frame=0, frame_interval=1, test_novel_pose=False)
    items = {}
    for steps in (None, "host", "device"):
        restore = _with_cfg(dict(base, **({} if steps is None else {"dataset_image_steps": steps})))
        try:
            cv = _Cv2Stub()
            items[steps] = make(cv)()[0]
            if steps == "device":
                assert "undistort" not in cv.calls and "resize" not in cv.calls
        finally:
            restore()
    host, dev = items["host"], items["device"]
    assert set(items[None]) == set(host) and all(np.array_equal(np.asarray(items[None][k]), np.asarray(host[k]))
                                                 for k in host if k != "meta")
    moved = {"img", "ray_class"} | ({"msk"} if kind == "mono" else set())
    added = {"img_u8", "msk_u8"} | ({"bound_mask"} if split == "train" else set())
    assert set(dev) == (set(host) - moved) | added
    for k in set(host) - moved - {"meta"}:
        assert np.array_equal(np.asarray(dev[k]), np.asarray(host[k])), k
    for k in host["meta"]:
        assert np.array_equal(np.asarray(dev["meta"][k]), np.asarray(host["meta"][k])), k
    assert np.array_equal(dev["img_u8"], img_u8) and np.array_equal(dev["msk_u8"], msk)
    m = dev["meta"]
    assert m["image_n_dist"] == 5 and m["image_size"].tolist() == [8, 6] and m["image_bkgd"] == 2
    assert m["image_msk"] == (kind == "mono") and m["image_cam"][:9].tolist() == K.ravel().tolist()
    assert m["image_cam"][9:14].tolist() == D.astype(np.float32 if kind == "mono" else np.float64).ravel().tolist()
    if split == "train":
        assert np.array_equal(dev["bound_mask"], bound)
        assert m["image_class"] == (train_item.CLASS_H36M if kind == "mv" else train_item.CLASS_SNAPSHOT)
    else:
        assert m["image_class"] == 0


@pytest.mark.parametrize("what", ["ratio", "size", "dist"])
def test_dropin_device_item_rejects_unsupported_geometry(what):
    from neuralbody_b200.lib.datasets.light_stage import multi_view_dataset as mv
    img_u8 = np.zeros((16, 12, 3), np.uint8)
    msk = np.ones((16, 12), np.uint8)
    K = np.array([[20., 0, 6], [0, 20, 8], [0, 0, 1]])
    D = np.zeros((6, 1)) if what == "dist" else np.zeros((5, 1))
    cfg = dict(H=16, W=12, ratio=0.25 if what == "ratio" else 0.5, mask_bkgd=True, white_bkgd=False,
               body_sample_ratio=0.5, face_sample_ratio=0.0, begin_ith_frame=0, frame_interval=1, test_novel_pose=False,
               dataset_image_steps="device")
    if what == "size":
        cfg.update(H=32, W=24)
    restore = _with_cfg(cfg)
    try:
        cls = mv.make_dataset_class(_mv_base("train", msk, K, D), cv2=_Cv2Stub(), imread=lambda p: img_u8.copy(),
                                    bound_2d_mask=lambda *a: np.ones((a[3], a[4]), np.uint8))
        with pytest.raises(ValueError):
            cls()[0]
    finally:
        restore()
