"""nb_image_rays / nb_image_rays_f64 argument validation and the demo dataset drop-ins, without a GPU."""
import ctypes as C

import numpy as np
import pytest

from tools import demo_case as DC


def lib():
    from neuralbody_b200 import capi
    return capi.load()


def args(H=4, W=5, ws=1 << 20):
    from neuralbody_b200 import capi
    a = capi.nb_image_rays_args()
    a.H, a.W = H, W
    a.workspace, a.workspace_bytes = 256, ws          # never dereferenced: validation fails before anything is enqueued
    a.ray_o = a.ray_d = a.near = a.far = a.mask_at_box = a.count = 256
    return a


def cam(ct):
    arrs = [(ct * 9)(*range(9)), (ct * 9)(*range(9)), (ct * 3)(1, 2, 3), (ct * 3)(1, 2, 3)]
    return [C.cast(x, C.POINTER(ct)) for x in arrs]


@pytest.mark.parametrize("name,ct", [("nb_image_rays", C.c_float), ("nb_image_rays_f64", C.c_double)])
def test_bad_arguments_are_rejected_before_any_launch(name, ct):
    L = lib()
    fn = getattr(L, name)
    K, R, T, o = cam(ct)
    null = C.cast(None, C.POINTER(ct))
    assert fn(None, K, R, T, o, None) == -1
    for i in range(4):
        ptrs = [K, R, T, o]
        ptrs[i] = null
        assert fn(C.byref(args()), *ptrs, None) == -1
    for field in ("workspace", "ray_o", "ray_d", "near", "far", "mask_at_box", "count"):
        a = args()
        setattr(a, field, None)
        assert fn(C.byref(a), K, R, T, o, None) == -1, field
        assert b"null" in L.nb_last_error()
    for H, W in ((0, 5), (5, 0), (-1, 3), (1 << 16, 1 << 15)):
        assert fn(C.byref(args(H, W)), K, R, T, o, None) == -1
        assert b"H and W" in L.nb_last_error()
    assert L.nb_image_rays_workspace_bytes(0, 4) == 0 and L.nb_image_rays_workspace_bytes(1 << 16, 1 << 15) == 0


@pytest.mark.parametrize("name,ct", [("nb_image_rays", C.c_float), ("nb_image_rays_f64", C.c_double)])
def test_short_workspace_is_rejected(name, ct):
    L = lib()
    need = L.nb_image_rays_workspace_bytes(48, 64)
    if need == 0:
        pytest.skip("the scan's scratch size needs a CUDA device to be queried")
    assert need >= 48 * 64 * 4
    assert getattr(L, name)(C.byref(args(48, 64, need - 1)), *cam(ct), None) == -1
    assert b"workspace_bytes too small" in L.nb_last_error()


def test_camera_dtype_and_shape_errors():
    from neuralbody_b200 import rays
    b = np.zeros((2, 3), np.float32)
    with pytest.raises(ValueError, match="float32 or all float64"):
        rays.camera_image_rays(np.eye(4), np.eye(3, dtype=np.float32), b, 4, 4)
    with pytest.raises(ValueError, match="float32 or all float64"):
        rays.camera_image_rays(np.eye(4, dtype=np.float16), np.eye(3, dtype=np.float16), b, 4, 4)
    with pytest.raises(ValueError, match="RT must be"):
        rays.camera_image_rays(np.eye(3), np.eye(3), b, 4, 4)
    with pytest.raises(ValueError, match="can_bounds"):
        rays.camera_image_rays(np.eye(4), np.eye(3), b.astype(np.float64), 4, 4)


@pytest.mark.parametrize("golden", [DC.GOLDEN_MV, DC.GOLDEN_MONO], ids=["float64", "float32"])
def test_restatement_reproduces_the_goldens(golden):
    """The numpy restatement the GPU tests compare against reproduces upstream's recorded output bit for bit."""
    g = DC.load_golden(golden)
    for v, c in g["views"].items():
        got = DC.image_rays_numpy(c["RT"], c["K"], c["bounds"], g["H"], g["W"])
        for k, x in zip(("ray_o", "ray_d", "near", "far", "mask_at_box"), got):
            assert np.array_equal(x, c[k]) and x.dtype == c[k].dtype, (v, k)


@pytest.mark.parametrize("golden", [DC.GOLDEN_MV, DC.GOLDEN_MONO], ids=["float64", "float32"])
def test_upstreams_plain_numpy_reproduces_the_goldens(golden):
    """The plain np.dot / np.linalg.norm computation tools/bench_demo.py times as upstream's host cost gives upstream's
    recorded output too."""
    g = DC.load_golden(golden)
    for v, c in g["views"].items():
        got = DC.upstream_image_rays(c["RT"], c["K"], c["bounds"], g["H"], g["W"])
        for k, x in zip(("ray_o", "ray_d", "near", "far", "mask_at_box"), got):
            assert np.array_equal(x, c[k]) and x.dtype == c[k].dtype, (v, k)


@pytest.mark.parametrize("which", ["mv", "mono", "orbit"])
def test_golden_inputs_match_their_checksum(which, tmp_path):
    """The synthetic data the goldens were generated from is rebuilt and hashed as the generator hashed it."""
    pytest.importorskip("cv2")
    d = str(tmp_path)
    if which == "mv":
        masks, want = DC.write_mv_root(d), DC.load_golden(DC.GOLDEN_MV)["input_sha256"]
    elif which == "mono":
        masks, want = DC.write_mono_root(d)[1], DC.load_golden(DC.GOLDEN_MONO)["input_sha256"]
    else:
        masks, want = DC.write_orbit_root(d)[1], bytes(np.load(DC.ORBIT)["input_sha256"]).decode()
    assert DC.input_checksum(d, masks) == want


def test_exact_fma_emulation():
    rng = np.random.RandomState(0)
    a, b = rng.randn(1000), rng.randn(1000)
    c = -(a * b)
    # a * b + c with c = -RN(a * b) is the product's rounding error, which the two-product gives exactly
    from tools.demo_case import _two_prod
    assert np.array_equal(DC.fma64(a, b, c), _two_prod(a, b)[1])
    a32, b32 = a.astype(np.float32), b.astype(np.float32)
    c32 = -(a32 * b32)
    err = (a32.astype(np.float64) * b32 + c32).astype(np.float32)   # exact in float64 and in float32
    assert np.array_equal(DC.fma32(a32, b32, c32), err)


# ----------------------------------------------------------------------------- dataset drop-ins (need the reference tree)
def _reference():
    from oracle import ref_harness
    if not ref_harness.reference_available():
        pytest.skip("the reference tree is not available")
    pytest.importorskip("cv2")


@pytest.mark.parametrize("kind,views", [("mv", (0, 37, 90)), ("perform", (0, 1)), ("mono", (0, 50))])
def test_dropin_item_is_upstreams_item_without_the_rays(kind, views, tmp_path):
    _reference()
    import importlib
    from neuralbody_b200.lib.config import cfg as nb_cfg
    pairs, _, ds, masks = DC.reference_items(kind, views, str(tmp_path))
    from oracle import ref_harness
    rcfg = ref_harness.load_reference()[0]
    for k in ("H", "W", "ratio", "ith_frame", "begin_ith_frame", "num_train_frame"):
        setattr(nb_cfg, k, rcfg[k])
    name = {"mv": "multi_view_demo_dataset", "perform": "multi_view_perform_dataset", "mono": "monocular_demo_dataset"}[kind]
    mod = importlib.import_module("neuralbody_b200.lib.datasets.light_stage." + name)
    kw = {"imread": lambda p: masks[p].copy()} if kind == "mono" else {}
    ref_mod = importlib.import_module(mod.REFERENCE_MODULE)
    import types
    old = ref_mod.imageio
    ref_mod.imageio = types.SimpleNamespace(imread=lambda p: masks[p].copy())
    try:
        cls = mod.make_dataset_class(type(ds), **kw)
        mine = cls.__new__(cls)
        mine.__dict__.update(ds.__dict__)
        for v, (item, call) in zip(views, pairs):
            got = mine[v]
            assert set(got) == (set(item) - {"ray_o", "ray_d", "near", "far", "mask_at_box"}) | {"cam_RT", "cam_K", "can_bounds",
                                                                                                 "meta"}
            assert set(got["meta"]) == {"cam_RT", "cam_K", "can_bounds"}
            assert all(got["meta"][k] is got[k] for k in got["meta"])
            for k in item:
                if k in ("ray_o", "ray_d", "near", "far", "mask_at_box"):
                    continue
                a, b = np.asarray(got[k]), np.asarray(item[k])
                assert a.dtype == b.dtype and np.array_equal(a, b), (kind, v, k)
            for k, ref_k in (("cam_RT", "RT"), ("cam_K", "K"), ("can_bounds", "bounds")):
                a = np.asarray(got[k])
                assert a.dtype == call[ref_k].dtype and np.array_equal(a, call[ref_k]), (kind, v, k)
    finally:
        ref_mod.imageio = old
