"""CPU: the numpy restatement of the demo and mesh datasets' mask views (tools/mask_views_case.py) against OpenCV, the
goldens, the drop-ins' `dataset_image_steps: 'device'` items and the validation that refuses what nb_mask_views does not
implement before any launch."""
import numpy as np
import pytest
import torch

from oracle import item_images as O
from tools import mask_views_case as MC

SIZES = [(1024, 1024), (1080, 1080), (1002, 1000)]
DISTS = ["d4", "d5", "rational8", "zero", "k1"]


@pytest.mark.parametrize("size", SIZES, ids=["%dx%d" % s for s in SIZES])
@pytest.mark.parametrize("dist", DISTS)
def test_restatement_equals_opencv(size, dist):
    """Every value set ({0,1}, {0,255}, arbitrary 0..255 unbinarised), binarised or not, dilation on and off, copy and
    2x: the restatement is OpenCV's output; pixels near a 1/32 px rounding tie are counted and may not differ either."""
    cv2 = pytest.importorskip("cv2")
    H0, W0 = size
    K, D = MC.camera(H0, W0, dist, H0 + W0)
    U, V = O.undistort_uv(K, D, H0, W0)
    tie = O.near_tie(U) | O.near_tie(V)
    for values in MC.VALUES:
        msk = MC.silhouette(H0, W0, values, H0 + len(values))
        for binarise in (False, True):
            src = (msk != 0).astype(np.uint8) if binarise else msk
            und = O.remap(src, U, V)
            assert np.array_equal(und, cv2.undistort(src, K, D)), (values, binarise)
            for dil in (0, 5):
                m = MC.dilate(und, dil)
                t = MC.dilate(tie.astype(np.uint8), dil).astype(bool)
                for k in (1, 2):
                    H, W = H0 // k, W0 // k
                    want = MC.cv2_mask_view(msk, K, D, H, W, binarise, dil)
                    got = m[::k, ::k]
                    print("%s %s %s bin=%d dil=%d k=%d: %d flagged pixels, %d of them differ"
                          % (size, dist, values, binarise, dil, k, t[::k, ::k].sum(), (got != want)[t[::k, ::k]].sum()))
                    assert np.array_equal(got, want), (values, binarise, dil, k)


def test_restatement_equals_the_goldens():
    for g in MC.load_golden():
        binarise, dil, _ = MC.RECIPES[g["recipe"]]
        H, W = g["msks"].shape[1:]
        for v in range(len(g["Ds"])):
            got, _ = MC.mask_view(g["msks_u8"][v], g["Ks"][v], g["Ds"][v], H, W, binarise, dil)
            assert np.array_equal(got, g["msks"][v]), (g["recipe"], v)


def test_goldens_are_opencvs():
    """tools/mask_views_case.py writes what cv2 computes today: regenerate and compare (needs OpenCV)."""
    pytest.importorskip("cv2")
    for c, g in enumerate(MC.load_golden()):
        recipe, H0, W0, ratio, dists, values, seed = MC.GOLDEN_CASES[c]
        msks_u8, Ks, Ds = MC.case(H0, W0, dists, values, seed)
        assert np.array_equal(msks_u8, g["msks_u8"]) and np.array_equal(Ks, g["Ks"])
        binarise, dil, _ = MC.RECIPES[recipe]
        H, W = MC.out_size(H0, W0, ratio)
        want = np.stack([MC.cv2_mask_view(m, K, D, H, W, binarise, dil) for m, K, D in zip(msks_u8, Ks, Ds)])
        assert np.array_equal(want, g["msks"]), recipe


# ----------------------------------------------------------------------------- the drop-ins' 'device' items
HOST_KEY = {"multi_view_demo": "msks", "multi_view_perform": "msks", "monocular_demo": "msk", "multi_view_mesh": "msks",
            "monocular_mesh": "msks"}


@pytest.mark.parametrize("kind", list(MC.DROP_INS))
def test_dropin_device_item(kind):
    """The 'device' item is the 'host' item with the processed masks replaced by the decoded ones (`msks_u8` (nv,H0,W0)
    uint8 as read, before any binarising) and the recipe under 'meta'; the restatement of that recipe is the host item's
    masks bit for bit."""
    pytest.importorskip("cv2")
    ratio = 1.0 if kind == "multi_view_mesh" else 0.5
    host, dev = MC.item_pair(kind, 40, 52, 3, ratio, seed=2, values="any")
    key = HOST_KEY[kind]
    assert set(dev) == (set(host) - {key}) | {"msks_u8", "meta"}
    for k in set(host) - {key, "meta"}:
        a, b = np.asarray(dev[k]), np.asarray(host[k])
        assert a.dtype == b.dtype and np.array_equal(a, b), k
    for k in host.get("meta", {}):
        assert np.array_equal(np.asarray(dev["meta"][k]), np.asarray(host["meta"][k])), k
    nv = 1 if kind in MC.MONOCULAR else 3
    m = dev["meta"]
    assert dev["msks_u8"].shape == (nv, 40, 52) and dev["msks_u8"].dtype == np.uint8
    assert len(np.unique(dev["msks_u8"])) > 2                  # as decoded: not binarised
    assert m["mask_cams"].shape == (nv, 17) and m["mask_cams"].dtype == np.float64
    assert m["mask_size"].tolist() == [int(40 * ratio), int(52 * ratio)] and m["mask_size"].dtype == np.int64
    assert (m["mask_binarise"], m["mask_dilate"]) == ((0, 0) if kind in MC.MONOCULAR else (1, 5))
    assert m["mask_n_dist"] == (8 if kind in MC.MONOCULAR else 5)
    want = np.asarray(host[key]).reshape(nv, *m["mask_size"].tolist())
    got, tie = MC.restate_item(dev)
    print("%s: %d flagged pixels" % (kind, tie.sum()))
    assert np.array_equal(got, want)


@pytest.mark.parametrize("what", ["rgb", "float", "sizes", "ratio", "dist", "wide"])
def test_unsupported_items_raise_value_error(what):
    """What nb_mask_views does not implement raises ValueError in the item, before any GPU work."""
    from neuralbody_b200.lib.datasets import mask_item
    m = np.zeros((16, 12), np.uint8)
    K, D = np.array([[20., 0, 6], [0, 20, 8], [0, 0, 1]]), np.zeros((5, 1))
    args = dict(msks_u8=[m, m], Ks=[K, K], Ds=[D, D], H=8, W=6, binarise=True, dilate=5)
    if what == "rgb":
        args["msks_u8"] = [np.zeros((16, 12, 3), np.uint8)] * 2
    elif what == "float":
        args["msks_u8"] = [m.astype(np.float32)] * 2
    elif what == "sizes":
        args["msks_u8"] = [m, np.zeros((16, 14), np.uint8)]
    elif what == "ratio":
        args.update(H=4, W=3)
    elif what == "dist":
        args["Ds"] = [D, np.zeros((6, 1))]
    else:
        args.update(msks_u8=[np.zeros((2, 4098), np.uint8)] * 2, H=1, W=2049)
    with pytest.raises(ValueError):
        mask_item.mask_fields(**args)


def test_dropin_item_raises_on_unsupported_ratio():
    pytest.importorskip("cv2")
    Base, imread, cfg = MC.stand_in("multi_view_demo", 40, 52, 2, 0.25)
    restore = MC.with_cfg(dict(cfg, dataset_image_steps="device"))
    try:
        with pytest.raises(ValueError):
            MC.make_item("multi_view_demo", Base, imread, 0)
    finally:
        restore()


def test_wrapper_validates_before_launch(built_lib):
    """images.mask_views refuses host tensors, wrong dtypes and shapes and unsupported recipes before any CUDA call;
    nb_mask_views itself refuses bad arguments without touching the device."""
    import ctypes
    from neuralbody_b200 import capi, images
    cams = np.zeros((2, capi.NB_ITEM_CAM_DOUBLES))
    with pytest.raises(ValueError):
        images.mask_views(torch.zeros((2, 16, 12), dtype=torch.uint8), cams, 5, 8, 6, 1, 5)
    lib = capi.load()
    a = capi.nb_mask_views_args()
    assert lib.nb_mask_views(ctypes.byref(a), None) < 0 and b"null" in lib.nb_last_error()
    a.msk_u8 = a.cams = a.msks = 1
    a.nv, a.H0, a.W0, a.H, a.W, a.n_dist = 2, 16, 12, 4, 3, 5
    assert lib.nb_mask_views(ctypes.byref(a), None) < 0 and b"half" in lib.nb_last_error()
    a.H, a.W, a.dilate = 8, 6, 5
    assert lib.nb_mask_views(ctypes.byref(a), None) < 0 and b"null" in lib.nb_last_error()     # a dilation's workspace
    a.dilate, a.workspace, a.workspace_bytes = 3, 1, 10
    assert lib.nb_mask_views(ctypes.byref(a), None) < 0 and b"dilate" in lib.nb_last_error()
    a.dilate = 5
    assert lib.nb_mask_views(ctypes.byref(a), None) < 0 and b"workspace" in lib.nb_last_error()
    assert lib.nb_mask_views_workspace_bytes(2, 16, 12) == 2 * 16 * 12 and lib.nb_mask_views_workspace_bytes(0, 1, 1) == 0
