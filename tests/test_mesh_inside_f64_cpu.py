"""CPU: the float64-camera mask test of the People-Snapshot mesh path without a GPU -- nb_mesh_inside_f64 refuses bad
arguments before it touches the device, its kernel compiles without spills, the renderer picks the projection by the
camera's dtype and refuses a mixed one, and the monocular dataset drop-in returns the mask view the reference's
prepare_inside_pts received (tests/golden/mesh_mono_s03.npz)."""
import ctypes
import hashlib
import os
import re
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from conftest import ROOT
from tools import mesh_mono_case as MM

MESH_RENDERER = os.path.join(ROOT, "neuralbody_b200", "lib", "networks", "renderer", "if_mesh_renderer.py")


def _ren_module():
    from neuralbody_b200.lib.networks.make_network import load_source
    return load_source("neuralbody_b200.lib.networks.renderer.if_mesh_renderer", MESH_RENDERER)


def test_mesh_inside_f64_rejects_bad_arguments(built_lib):
    """Every refusal returns before a CUDA call (the pointers are never dereferenced)."""
    from neuralbody_b200 import capi
    lib = capi.load()
    fake = 256                                     # non-null, never read

    def args(**kw):
        a = capi.nb_mesh_inside_args()
        a.x = a.y = a.z = a.msks = a.inside = fake
        a.RT = a.Ks = None
        a.nx, a.ny, a.nz, a.nv, a.H, a.W = 4, 5, 6, 1, 8, 9
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    def call(a, RT=fake, Ks=fake):
        return lib.nb_mesh_inside_f64(None if a is None else ctypes.byref(a), RT, Ks, None)

    assert call(None) == -1 and b"null" in lib.nb_last_error()
    for k in ("x", "y", "z", "msks", "inside"):
        assert call(args(**{k: None})) == -1, k
        assert b"nb_mesh_inside_f64: null" in lib.nb_last_error()
    assert call(args(), RT=None) == -1 and b"null" in lib.nb_last_error()
    assert call(args(), Ks=None) == -1 and b"null" in lib.nb_last_error()
    for k in ("RT", "Ks"):                          # the float32 camera's fields must stay empty
        assert call(args(**{k: fake})) == -1, k
        assert b"must be NULL" in lib.nb_last_error()
    for k in ("nv", "H", "W"):
        for v in (0, -1):
            assert call(args(**{k: v})) == -1, (k, v)
            assert b"nb_mesh_inside_f64: nv, H and W must be >= 1" in lib.nb_last_error()
    for k in ("nx", "ny", "nz"):
        assert call(args(**{k: 0})) == -1, k
        assert b"grid dims" in lib.nb_last_error()
    assert call(args(nx=1291, ny=1291, nz=1291)) == -2          # 1291^3 > 2^31 points
    assert b"2^31" in lib.nb_last_error()
    # the float32 entry point still requires its camera in the struct
    a = args()
    assert lib.nb_mesh_inside(ctypes.byref(a), None) == -1 and b"nb_mesh_inside: null" in lib.nb_last_error()


def test_mesh_inside_f64_kernel_has_no_spills(tmp_path):
    from neuralbody_b200 import _build
    src = os.path.join(ROOT, "neuralbody_b200", "csrc", "nb_mesh_inside_f64.cu")
    cmd = [_build.find_nvcc()] + _build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", "-o", str(tmp_path / "f64.o"), src]
    log = subprocess.run(cmd, capture_output=True, text=True, check=True).stderr
    entries = [e for e in log.split("Compiling entry function")[1:] if "mesh_inside_kernel" in e.split("\n")[0]]
    assert len(entries) == 1 and "mesh_inside_kernelId" in entries[0].split("\n")[0], log
    m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", entries[0])
    assert m and m.group(1) == "0" and m.group(2) == "0", entries[0]


def test_projection_follows_the_camera_dtype():
    ren = _ren_module()
    f32, f64 = torch.zeros(1, 3, 4), torch.zeros(1, 3, 4, dtype=torch.float64)
    assert ren.camera_is_f64(f64, f64[:, :, :3]) is True
    assert ren.camera_is_f64(f32, f32[:, :, :3]) is False
    with pytest.raises(ValueError, match="float64"):
        ren.camera_is_f64(f64, f32[:, :, :3])
    with pytest.raises(ValueError, match="float64"):
        ren.camera_is_f64(f32, f64[:, :, :3])
    # a mixed batch is refused before anything looks at the device
    r = ren.Renderer.__new__(ren.Renderer)
    mb = {"wbounds": torch.zeros(1, 2, 3), "RT": f64[None], "Ks": torch.eye(3)[None, None], "msks": torch.ones(1, 1, 4, 4, dtype=torch.uint8)}
    with pytest.raises(ValueError, match="RT and Ks"):
        r.grid_from_masks(mb)
    with pytest.raises(ValueError, match="RT and Ks"):
        r.grid_from_masks(dict(mb, RT=f32[None], Ks=torch.eye(3, dtype=torch.float64)[None, None]))


def test_golden_is_the_case_and_the_host_test():
    """The golden's inputs are this case's, its grid is world_axes', and its inside is the float64 restatement's."""
    gold = MM.load_golden()
    case = MM.build_case("mono_s03")
    assert MM.case_checksum(*case) == gold["input_sha256"]
    scene = case[0]
    axes = _ren_module().world_axes(scene["can_bounds"][0].numpy(), scene["voxel_size"])
    pts = np.stack(np.meshgrid(*axes, indexing="ij"), axis=-1)
    assert hashlib.sha256(np.ascontiguousarray(pts).tobytes()).hexdigest() == gold["pts_sha256"]
    assert gold["K"].dtype == gold["R"].dtype == gold["T"].dtype == np.float64
    np.testing.assert_array_equal(MM.mesh_inside_f64(pts, gold["K"], gold["R"], gold["T"], gold["msk"]), gold["inside"])
    # what the float64 camera is for: the same test with the camera cast to float32 reads other pixels
    f32 = MM.mesh_inside_f64(pts, gold["K"].astype(np.float32), gold["R"].astype(np.float32),
                             gold["T"].astype(np.float32), gold["msk"])
    print("camera cast to float32: %d of %d points read another value" % (int((f32 != gold["inside"]).sum()), f32.size))


@pytest.fixture(scope="module")
def dropin_item(tmp_path_factory):
    """The drop-in's item for the golden frame, built with OpenCV in a process of its own."""
    out = tmp_path_factory.mktemp("mono") / "item.npz"
    env = dict(os.environ, PYTHONNOUSERSITE="1")
    subprocess.run([sys.executable, "-m", "tools.mesh_mono_case", "--drop-in", str(out)], cwd=ROOT, env=env, check=True,
                   timeout=600)
    z = np.load(out)
    return {k: z[k] for k in z}


def test_dataset_drop_in_returns_the_mask_view(dropin_item):
    item, gold = dropin_item, MM.load_golden()
    scene = MM.build_case("mono_s03")[0]
    # the reference item's keys (monocular_mesh_dataset.py:91-104) without pts / inside, plus wbounds and the mask view
    assert set(item) == {"coord", "out_sh", "wbounds", "bounds", "R", "Th", "latent_index", "frame_index", "msks", "Ks", "RT"}
    assert np.array_equal(item["coord"], scene["coord"][0].numpy()) and np.array_equal(item["out_sh"], scene["out_sh"][0].numpy())
    assert item["wbounds"].dtype == np.float32 and np.array_equal(item["wbounds"], scene["can_bounds"][0].numpy())
    assert np.array_equal(item["bounds"], scene["bounds"][0].numpy())
    assert item["R"].dtype == np.float32 and np.allclose(item["R"], scene["R"][0].numpy(), atol=1e-6)
    assert int(item["latent_index"]) == 0 and int(item["frame_index"]) == 0
    # exactly what the reference's prepare_inside_pts received: the undistorted, resized mask and the float64 camera
    assert item["msks"].dtype == np.uint8 and np.array_equal(item["msks"], gold["msk"][None])
    assert item["Ks"].dtype == np.float64 and np.array_equal(item["Ks"], gold["K"][None])
    assert item["RT"].dtype == np.float64 and np.array_equal(item["RT"], np.concatenate([gold["R"], gold["T"]], axis=1)[None])


def test_dataset_drop_in_keeps_upstreams_indices():
    """latent_index is the item index, unclamped (num_train_frame = 1 here), frame_index adds begin_ith_frame; the mask is
    read from <data_root>/mask/<frame>.png.  OpenCV is replaced by a stand-in (identity undistortion, nearest resize)."""
    scene, pkl, msk, img = MM.build_case("mono_s03")
    paths = []

    def imread(path):
        paths.append(path)
        return msk.copy()

    def resize(m, wh, interpolation):
        ys = (np.arange(wh[1]) * m.shape[0]) // wh[1]
        xs = (np.arange(wh[0]) * m.shape[1]) // wh[0]
        return m[ys][:, xs]

    cv = types.SimpleNamespace(undistort=lambda m, K, D: m, resize=resize, INTER_NEAREST=0,
                               Rodrigues=lambda r: (MM.synth._rodrigues(r), None))
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.networks.make_network import load_source
    mod = load_source("neuralbody_b200.lib.datasets.light_stage.monocular_mesh_dataset",
                      os.path.join(ROOT, "neuralbody_b200", "lib", "datasets", "light_stage", "monocular_mesh_dataset.py"))
    Base = MM.stand_in_base(scene, pkl)

    class Later(Base):
        def __init__(self):
            super().__init__()
            self.begin_ith_frame = 3

    old = cfg.ratio
    cfg.ratio = 0.5
    try:
        it = mod.make_dataset_class(Later, cv2=cv, imread=imread)()[5]
    finally:
        cfg.ratio = old
    assert it["latent_index"] == 5 and it["frame_index"] == 8
    assert paths == [os.path.join("synthetic", "mask", "8.png")]
    assert it["msks"].shape == (1, 100, 75) and np.array_equal(it["msks"][0], resize(msk, (75, 100), 0))
    K = MM.get_camera(pkl)["K"]
    assert np.array_equal(it["Ks"][0, :2], K[:2] * 0.5) and np.array_equal(it["Ks"][0, 2], K[2])
