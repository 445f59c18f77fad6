"""CPU: the pieces of the mesh renderer's mask-view path that need no GPU -- the grid axes built on the host reproduce the
reference dataset's grid (tests/golden/mesh_s03.npz), nb_mesh_inside refuses bad arguments before it touches the device,
its kernel compiles without spills, and the dataset drop-in returns the mask views instead of `pts` / `inside`."""
import ctypes
import hashlib
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from oracle import mesh_case, synth

MESH_RENDERER = os.path.join(ROOT, "neuralbody_b200", "lib", "networks", "renderer", "if_mesh_renderer.py")
MESH_DATASET = os.path.join(ROOT, "neuralbody_b200", "lib", "datasets", "light_stage", "multi_view_mesh_dataset.py")


def _module(name, path):
    from neuralbody_b200.lib.networks.make_network import load_source
    return load_source(name, path)


def test_host_axes_reproduce_the_reference_grid():
    gold = mesh_case.load_golden()
    scene, _, _ = mesh_case.build_case("mesh_s03")
    ren = _module("neuralbody_b200.lib.networks.renderer.if_mesh_renderer", MESH_RENDERER)
    axes = ren.world_axes(scene["can_bounds"][0].numpy(), scene["voxel_size"])
    assert all(a.dtype == np.float32 and a.ndim == 1 for a in axes)
    assert tuple(len(a) for a in axes) == gold["shape"]
    pts = np.stack(np.meshgrid(*axes, indexing="ij"), axis=-1)
    assert hashlib.sha256(np.ascontiguousarray(pts).tobytes()).hexdigest() == gold["pts_sha256"]
    # the full-size grid: the axes are the dataset grid's planes
    full = synth.make_scene(**mesh_case.CASES["mesh_full"][0])
    cb, vs = full["can_bounds"][0].numpy(), full["voxel_size"]
    axes = ren.world_axes(cb, vs)
    assert tuple(len(a) for a in axes) == (170, 325, 146)
    for a in range(3):
        ref = np.arange(cb[0, a], cb[1, a] + vs[a], vs[a]).astype(np.float32)     # multi_view_mesh_dataset.py:151-156
        assert np.array_equal(axes[a].view(np.int32), ref.view(np.int32))


def test_mesh_inside_rejects_bad_arguments(built_lib):
    """Every refusal returns before a CUDA call (the pointers are never dereferenced)."""
    from neuralbody_b200 import capi
    lib = capi.load()
    fake = 256                                     # non-null, never read

    def args(**kw):
        a = capi.nb_mesh_inside_args()
        a.x = a.y = a.z = a.msks = a.RT = a.Ks = a.inside = fake
        a.nx, a.ny, a.nz, a.nv, a.H, a.W = 4, 5, 6, 2, 8, 9
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    assert lib.nb_mesh_inside(None, None) == -1 and b"null" in lib.nb_last_error()
    for k in ("x", "y", "z", "msks", "RT", "Ks", "inside"):
        assert lib.nb_mesh_inside(ctypes.byref(args(**{k: None})), None) == -1, k
        assert b"null" in lib.nb_last_error()
    for k in ("nv", "H", "W"):
        for v in (0, -1):
            assert lib.nb_mesh_inside(ctypes.byref(args(**{k: v})), None) == -1, (k, v)
            assert b">= 1" in lib.nb_last_error()
    for k in ("nx", "ny", "nz"):
        assert lib.nb_mesh_inside(ctypes.byref(args(**{k: 0})), None) == -1, k
        assert b"grid dims" in lib.nb_last_error()
    # 1291^3 = 2.15e9 > 2^31 points
    assert lib.nb_mesh_inside(ctypes.byref(args(nx=1291, ny=1291, nz=1291)), None) == -2
    assert b"2^31" in lib.nb_last_error()


def test_mesh_inside_kernel_has_no_spills(tmp_path):
    from neuralbody_b200 import _build
    src = os.path.join(ROOT, "neuralbody_b200", "csrc", "nb_mcubes.cu")
    cmd = [_build.find_nvcc()] + _build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", "-o", str(tmp_path / "mc.o"), src]
    log = subprocess.run(cmd, capture_output=True, text=True, check=True).stderr
    entries = [e for e in log.split("Compiling entry function")[1:] if "mesh_inside_kernel" in e.split("\n")[0]]
    assert len(entries) == 1, log
    m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", entries[0])
    assert m and m.group(1) == "0" and m.group(2) == "0", entries[0]


RH, TH = np.array([[0.3, -0.2, 0.1]]), np.array([[0.1, 0.2, 1.0]], np.float32)     # synth.make_scene's defaults


def stand_in_base(scene, masks):
    """The reference Dataset's attributes as its __init__ / prepare_input / get_mask leave them, for the synthetic scene
    (mesh_case._reference_item drives the reference's own methods on the same stand-in values)."""
    Ks, Rs, Ts, msks = mesh_case._views(masks)
    world = scene["verts_world"].numpy()

    class Base:
        def __init__(self):
            self.ims = np.zeros((1, len(msks)))
            self.Ks, self.Rs, self.Ts = Ks, Rs, Ts

        def prepare_input(self, i):
            coord, out_sh, can_bounds, bounds, _, Th = synth.prepare_input(world, RH.ravel(), TH.ravel(), scene["voxel_size"])
            return coord, out_sh, can_bounds, bounds, RH, TH

        def get_mask(self, i, nv):
            return msks[nv]

    return Base


def dataset_item(scene, masks, index=0):
    from neuralbody_b200.lib.config import cfg
    mod = _module("neuralbody_b200.lib.datasets.light_stage.multi_view_mesh_dataset", MESH_DATASET)
    cfg.num_train_frame = int(scene["weights"]["latent.weight"].shape[0])
    cfg.begin_ith_frame = 0
    # synth's restatement of cv2.Rodrigues, so that the test process does not load OpenCV (its own thread pools and BLAS)
    cls = mod.make_dataset_class(stand_in_base(scene, masks), rodrigues=lambda r: (synth._rodrigues(r), None))
    return cls()[index]


def test_dataset_drop_in_returns_the_mask_views():
    scene, masks, _ = mesh_case.build_case("mesh_s03")
    item = dataset_item(scene, masks)
    # the reference item's keys (multi_view_mesh_dataset.py:162-179) without pts / inside, plus the mask views
    assert set(item) == {"coord", "out_sh", "wbounds", "bounds", "R", "Th", "latent_index", "frame_index", "msks", "Ks", "RT"}
    assert np.array_equal(item["coord"], scene["coord"][0].numpy()) and np.array_equal(item["out_sh"], scene["out_sh"][0].numpy())
    assert item["wbounds"].dtype == np.float32 and np.array_equal(item["wbounds"], scene["can_bounds"][0].numpy())
    assert np.array_equal(item["bounds"], scene["bounds"][0].numpy())
    assert item["R"].dtype == np.float32 and np.allclose(item["R"], scene["R"][0].numpy(), atol=1e-6)
    assert item["latent_index"] == 0 and item["frame_index"] == 0
    Ks, Rs, Ts, msks = mesh_case._views(masks)
    nv = len(msks)
    assert item["msks"].dtype == np.uint8 and item["msks"].shape == (nv, 96, 96) and np.array_equal(item["msks"], msks)
    assert item["Ks"].dtype == np.float32 and np.array_equal(item["Ks"], Ks)
    assert item["RT"].dtype == np.float32 and item["RT"].shape == (nv, 3, 4)
    for v in range(nv):                                                       # prepare_inside_pts :126
        assert np.array_equal(item["RT"][v], np.concatenate([Rs[v], Ts[v]], axis=1))
    # the host test on the item's views and grid is the reference's inside (the golden)
    ren = _module("neuralbody_b200.lib.networks.renderer.if_mesh_renderer", MESH_RENDERER)
    pts = np.stack(np.meshgrid(*ren.world_axes(item["wbounds"], scene["voxel_size"]), indexing="ij"), axis=-1)
    inside = mesh_case.mesh_inside(pts, item["Ks"], item["RT"][:, :, :3], item["RT"][:, :, 3:], item["msks"])
    assert np.array_equal(inside, mesh_case.load_golden()["inside"])
