"""nb_train_rays argument validation, the restatement of upstream's training item, and the training dataset drop-ins,
without a GPU."""
import os
import types

import numpy as np
import pytest

from tools import train_rays_case as TC
from neuralbody_b200.lib.datasets import train_item


def lib():
    from neuralbody_b200 import capi
    return capi.load()


def args(B=1, H=4, W=5, n_rays=16, ws=1 << 20):
    from neuralbody_b200 import capi
    a = capi.nb_train_rays_args()
    a.B, a.H, a.W, a.n_rays = B, H, W, n_rays
    a.body_ratio, a.face_ratio = 0.5, 0.0
    a.k_kind, a.rt_kind = capi.NB_SCALAR_F64, capi.NB_SCALAR_F64
    a.workspace, a.workspace_bytes = 256, ws           # never dereferenced: validation fails before anything is enqueued
    a.class_map = a.image = a.cams = a.ray_o = a.ray_d = a.near = a.far = a.rgb = a.status = 256
    return a


def test_bad_arguments_are_rejected_before_any_launch():
    import ctypes as C
    L = lib()
    assert L.nb_train_rays(None, None) == -1
    for field in ("class_map", "image", "cams", "workspace", "ray_o", "ray_d", "near", "far", "rgb", "status"):
        a = args()
        setattr(a, field, None)
        assert L.nb_train_rays(C.byref(a), None) == -1, field
        assert b"null" in L.nb_last_error()
    a = args()
    a.draws = 256
    assert L.nb_train_rays(C.byref(a), None) == -1 and b"draw_offset" in L.nb_last_error()
    for B, H, W in ((0, 4, 4), (1, 0, 5), (1, 5, 0), (2, 1 << 15, 1 << 15)):
        assert L.nb_train_rays(C.byref(args(B, H, W)), None) == -1
        assert b"B, H and W" in L.nb_last_error()
    assert L.nb_train_rays(C.byref(args(n_rays=0)), None) == -1 and b"n_rays" in L.nb_last_error()
    for rb, rf in ((-0.1, 0.0), (0.7, 0.5), (float("nan"), 0.0)):
        a = args()
        a.body_ratio, a.face_ratio = rb, rf
        assert L.nb_train_rays(C.byref(a), None) == -1 and b"ratios" in L.nb_last_error()
    for kk, rk in ((2, 1), (0, 0), (1, 0)):
        a = args()
        a.k_kind, a.rt_kind = kk, rk
        assert L.nb_train_rays(C.byref(a), None) == -1 and b"k_kind" in L.nb_last_error()
    assert L.nb_train_rays_workspace_bytes(0, 4, 4) == 0 and L.nb_train_rays_workspace_bytes(2, 1 << 15, 1 << 15) == 0


def test_short_workspace_is_rejected():
    import ctypes as C
    L = lib()
    need = L.nb_train_rays_workspace_bytes(2, 48, 64)
    if need == 0:
        pytest.skip("the scan's scratch size needs a CUDA device to be queried")
    assert need >= 6 * 2 * 48 * 64 * 4
    assert L.nb_train_rays(C.byref(args(2, 48, 64, ws=need - 1)), None) == -1
    assert b"workspace_bytes too small" in L.nb_last_error()


@pytest.mark.parametrize("golden", [TC.GOLDEN_MV, TC.GOLDEN_MONO], ids=["multi_view", "monocular"])
def test_restatement_reproduces_the_goldens(golden):
    """The numpy restatement the GPU tests compare against reproduces upstream's recorded items bit for bit, from
    upstream's draws."""
    g = TC.load_golden(golden)
    assert max(int(it["rounds"]) for it in g["items"]) >= 2
    for c, (case, it) in enumerate(zip(g["cases"], g["items"])):
        got = TC.sample_numpy(it["img"], it["class_map"], it["K"], it["R"], it["T"], it["bounds"], case[1], case[2], case[3],
                              it["draws"])
        for k, x in zip(("rgb", "ray_o", "ray_d", "near", "far", "coord"), got):
            assert x.dtype == it[k].dtype and np.array_equal(x, it[k]), (c, k)
        assert got[6] == int(it["rounds"])


@pytest.mark.parametrize("golden", [TC.GOLDEN_MV, TC.GOLDEN_MONO], ids=["multi_view", "monocular"])
def test_upstreams_plain_numpy_reproduces_the_goldens(golden):
    """upstream_sample (what tools/bench_train_data.py times as upstream's host cost) gives upstream's items too, from the
    same np.random state."""
    g = TC.load_golden(golden)
    for c, (case, it) in enumerate(zip(g["cases"], g["items"])):
        rec = []
        orig = np.random.randint

        def replay(lo, hi, n):
            k = sum(len(r) for r in rec)
            rec.append(it["draws"][k:k + n])
            return rec[-1]
        np.random.randint = replay
        try:
            got = TC.upstream_sample(it["img"], it["class_map"], it["K"], it["R"], it["T"], it["bounds"], case[1], case[2],
                                     case[3])
        finally:
            np.random.randint = orig
        for k, x in zip(("rgb", "ray_o", "ray_d", "near", "far"), got):
            assert np.array_equal(x, it[k]), (c, k)


def test_value_error_conditions_match_upstreams():
    cm = np.zeros((4, 5), np.uint8)
    with pytest.raises(ValueError):
        train_item.check_lists(cm, 100, 0.5, 0.0)
    cm[1, 1] = train_item.BOUND
    with pytest.raises(ValueError):                 # body draws from an empty body list
        train_item.check_lists(cm, 100, 0.5, 0.0)
    train_item.check_lists(cm, 100, 0.0, 0.0)       # randint(0, 0, 0) does not raise
    train_item.check_lists(cm, 1, 0.5, 0.0)         # int(1 * 0.5) == 0 body draws
    cm[1, 1] |= train_item.BODY
    train_item.check_lists(cm, 100, 0.5, 0.3)       # an empty face list is skipped, as upstream
    for n, rb in ((100, 0.5), (1, 0.5), (100, 0.0)):   # numpy's own verdict for the same sizes
        for empty_body in (True, False):
            try:
                np.random.RandomState(0).randint(0, 0 if empty_body else 1, int(n * rb))
                want = False
            except ValueError:
                want = True
            m = np.full((2, 2), train_item.BOUND, np.uint8)
            if not empty_body:
                m[0, 0] |= train_item.BODY
            try:
                train_item.check_lists(m, n, rb, 0.0)
                got = False
            except ValueError:
                got = True
            assert got == want, (n, rb, empty_body)


def test_class_maps_follow_the_two_samplers():
    msk = np.array([[0, 1, 100, 13], [1, 1, 0, 13]], np.uint8)
    bm = np.array([[1, 1, 1, 1], [0, 1, 1, 1]], np.uint8)
    h = train_item.class_map_h36m(msk, bm)
    s = train_item.class_map_snapshot(msk, bm)
    B, F, O = train_item.BODY, train_item.FACE, train_item.BOUND
    assert h.tolist() == [[O, B | O, 0, F | O], [0, B | O, O, F | O]]          # border (100) out of the bound list
    assert s.tolist() == [[O, B | O, B | O, B | F | O], [0, B | O, O, B | F | O]]


# ----------------------------------------------------------------------------- dataset drop-ins over a stand-in base
class _Cv2Stub:
    """Records the drop-in's OpenCV calls; resize and undistort hand back the image at the requested size (nearest pixel),
    so the test sees which array went where."""
    INTER_AREA, INTER_NEAREST = 3, 0

    def __init__(self):
        self.calls = []

    def resize(self, a, size, interpolation=None):
        self.calls.append(("resize", a.dtype, size, interpolation))
        W, H = size
        ys = np.arange(H) * a.shape[0] // H
        xs = np.arange(W) * a.shape[1] // W
        return a[ys][:, xs].copy()

    def undistort(self, a, K, D):
        self.calls.append(("undistort", a.dtype))
        return a.copy()

    def Rodrigues(self, r):
        return (np.eye(3), None)


def _mv_base(split, img_u8, msk, K):
    class Base:
        def __init__(self):
            self.data_root, self.human, self.split, self.nrays = "/data", "CoreView_377", split, 500
            self.ims, self.cam_inds = np.array(["Camera_B1/000003.jpg"]), np.array([0])
            self.cams = {"K": [K], "D": [np.zeros((5, 1))], "R": [np.eye(3)], "T": [np.array([[0.], [0.], [2000.]])]}

        def get_mask(self, index):
            return msk.copy()

        def prepare_input(self, i):
            assert i == 3
            cb = np.array([[-0.5, -0.5, 1.5], [0.5, 0.5, 2.5]], np.float32)
            return (np.zeros((4, 3), np.int32), np.array([32, 32, 32], np.int32), cb, cb.copy(), np.zeros((1, 3)),
                    np.zeros((1, 3), np.float32))

        def __getitem__(self, index):
            return {"upstream": index}
    return Base


@pytest.mark.parametrize("split", ["train", "test"])
def test_dropin_item_over_a_stand_in_base(split):
    """multi_view_dataset's drop-in over a base with the reference's attributes, without the reference tree: upstream's
    image steps in upstream's order, the background, the class map of the bound mask it is handed, the camera of
    train_camera and, for split 'train', upstream's ValueError on an empty body list."""
    from neuralbody_b200.lib.config import get_active_cfg
    from neuralbody_b200.lib.datasets.light_stage import multi_view_dataset as mv
    from neuralbody_b200 import rays
    rng = np.random.RandomState(0)
    img_u8 = rng.randint(0, 256, (16, 12, 3)).astype(np.uint8)
    msk = np.zeros((16, 12), np.uint8)
    msk[4:12, 3:9] = 1
    msk[4, 3:9] = 100
    K = np.array([[20., 0, 6], [0, 20, 8], [0, 0, 1]])
    bound = np.zeros((8, 6), np.uint8)
    bound[1:7, 1:5] = 1
    seen = {}

    def b2d(cb, Kb, pose, H, W):
        seen.update(K=Kb.copy(), pose=pose.copy(), HW=(H, W))
        return bound.copy()
    cv = _Cv2Stub()
    cfg = get_active_cfg()          # the reference's config when its lib.config is loaded, as the drop-in reads it
    new = dict(H=16, W=12, ratio=0.5, mask_bkgd=True, white_bkgd=False, body_sample_ratio=0.5, face_sample_ratio=0.0,
               begin_ith_frame=0, frame_interval=1, test_novel_pose=False)
    old = {k: cfg[k] for k in new if k in cfg}
    dict.update(cfg, new)
    try:
        cls = mv.make_dataset_class(_mv_base(split, img_u8, msk, K), cv2=cv, imread=lambda p: img_u8.copy(),
                                    bound_2d_mask=b2d)
        item = cls()[0]
        small = cv.resize(msk, (6, 8))
        want = cv.resize(img_u8.astype(np.float32) / 255., (6, 8))
        want[small == 0] = 0
        assert item["img"].dtype == np.float32 and np.array_equal(item["img"], want)
        assert [c[0] for c in cv.calls[:5]] == ["resize", "undistort", "undistort", "resize", "resize"]
        assert not set(train_item.RAY_KEYS) & set(item)
        Ks = K.copy()
        Ks[:2] *= 0.5
        kind, cam = rays.train_camera(Ks, np.eye(3), np.array([[0.], [0.], [2.]]), item["can_bounds"])
        assert kind == 1 and np.array_equal(item["train_cam"], cam) and np.array_equal(item["meta"]["train_cam"], cam)
        assert item["frame_index"] == 3 and item["latent_index"] == 3 and item["cam_ind"] == 0
        if split == "train":
            assert np.array_equal(item["ray_class"], train_item.class_map_h36m(small, bound))
            assert np.array_equal(seen["K"], Ks) and seen["HW"] == (8, 6)
            assert item["meta"]["N_rand"] == 500 and item["meta"]["body_sample_ratio"] == 0.5
            with pytest.raises(ValueError):
                cls2 = mv.make_dataset_class(_mv_base(split, img_u8, np.zeros_like(msk), K), cv2=_Cv2Stub(),
                                             imread=lambda p: img_u8.copy(), bound_2d_mask=b2d)
                cls2()[0]
        else:
            assert "ray_class" not in item and set(item["meta"]) == {"train_cam", "train_k_kind", "can_bounds"}
    finally:
        for k in new:
            dict.pop(cfg, k, None)
        dict.update(cfg, old)


# ----------------------------------------------------------------------------- dataset drop-ins (need the reference tree)
def _reference():
    from oracle import ref_harness
    if not ref_harness.reference_available():
        pytest.skip("the reference tree is not available")
    pytest.importorskip("cv2")


@pytest.mark.parametrize("kind", ["mv", "mono"])
def test_dropin_test_split_is_upstreams_item_without_the_rays(kind, tmp_path):
    """Split 'test': upstream's keys minus the six ray keys, the image upstream's sampler received, and the camera."""
    _reference()
    import importlib
    pairs, _, ds, files = TC.reference_items(kind, ((TC.TEST_INDEX, 1024, 0.5, 0.0, False),), str(tmp_path), "test")
    name = "multi_view_dataset" if kind == "mv" else "monocular_dataset"
    mod = importlib.import_module("neuralbody_b200.lib.datasets.light_stage." + name)
    ref_mod = importlib.import_module(mod.REFERENCE_MODULE)
    read = lambda p: files[p].copy()
    old = ref_mod.imageio
    ref_mod.imageio = types.SimpleNamespace(imread=read)
    try:
        cls = mod.make_dataset_class(type(ds), imread=read, bound_2d_mask=ref_mod.if_nerf_dutils.get_bound_2d_mask)
        mine = cls.__new__(cls)
        mine.__dict__.update(ds.__dict__)
        got = mine[TC.TEST_INDEX]
    finally:
        ref_mod.imageio = old
    (item, call), = pairs
    assert set(got) == (set(item) - set(train_item.RAY_KEYS)) | {"img", "train_cam", "can_bounds", "meta"}
    for k in set(item) - set(train_item.RAY_KEYS):
        a, b = np.asarray(got[k]), np.asarray(item[k])
        assert a.dtype == b.dtype and np.array_equal(a, b), (kind, k)
    assert np.array_equal(got["img"], call["img"]) and np.array_equal(got["can_bounds"], call["bounds"])


@pytest.mark.parametrize("kind", ["mv", "mono"])
def test_dropin_item_is_upstreams_item_without_the_rays(kind, tmp_path):
    """The drop-in over the reference's Dataset: upstream's keys minus the six ray keys, the same image and mask as
    upstream's sampler received, and the class map of upstream's own bound mask."""
    _reference()
    import importlib
    from neuralbody_b200.lib.config import cfg as nb_cfg
    cases = TC.MV_CASES if kind == "mv" else TC.MONO_CASES
    pairs, _, ds, files = TC.reference_items(kind, cases, str(tmp_path))
    from oracle import ref_harness
    rcfg = ref_harness.load_reference()[0]
    name = "multi_view_dataset" if kind == "mv" else "monocular_dataset"
    mod = importlib.import_module("neuralbody_b200.lib.datasets.light_stage." + name)
    ref_mod = importlib.import_module(mod.REFERENCE_MODULE)
    d = str(tmp_path)
    for (index, nrays, rb, rf, face), (item, call) in zip(cases, pairs):
        rcfg.body_sample_ratio, rcfg.face_sample_ratio = rb, rf
        alias = {os.path.join(d, "mask", "0.png"): os.path.join(d, "mask13", "0.png")} if face else {}
        read = lambda p: files[alias.get(p, p)].copy()
        old = ref_mod.imageio
        ref_mod.imageio = types.SimpleNamespace(imread=read)
        try:
            cls = mod.make_dataset_class(type(ds), imread=read, bound_2d_mask=ref_mod.if_nerf_dutils.get_bound_2d_mask)
            mine = cls.__new__(cls)
            mine.__dict__.update(ds.__dict__)
            mine.nrays = nrays
            got = mine[index]
        finally:
            ref_mod.imageio = old
        extra = {"img", "ray_class", "train_cam", "can_bounds", "meta"}
        assert set(got) == (set(item) - set(train_item.RAY_KEYS)) | extra
        for k in set(item) - set(train_item.RAY_KEYS):
            a, b = np.asarray(got[k]), np.asarray(item[k])
            assert a.dtype == b.dtype and np.array_equal(a, b), (kind, index, k)
        assert got["img"].dtype == np.float32 and np.array_equal(got["img"], call["img"])
        assert np.array_equal(got["ray_class"], TC.class_map_of(kind, call))
        assert np.array_equal(got["can_bounds"], call["bounds"])
        assert got["meta"]["N_rand"] == nrays and got["meta"]["face_sample_ratio"] == rf
    assert nb_cfg is not None
