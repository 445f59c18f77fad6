"""GPU: the marching-cubes kernels (nb_mcubes_count / nb_mcubes_emit) against the numpy restatement, bit for bit, and the
mesh renderer (the drop-in for if_mesh_renderer.py) against the cube the unmodified reference built (tests/golden/
mesh_s03.npz)."""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import mcubes_oracle as M
from oracle import mesh_case
import gpu_utils as G
from test_mcubes_cpu import _smooth_field, ball_field, tie_field

pytestmark = pytest.mark.gpu

MESH_RENDERER = os.path.join(ROOT, "neuralbody_b200", "lib", "networks", "renderer", "if_mesh_renderer.py")


def _gpu_mc(vol, iso):
    from neuralbody_b200.mcubes import marching_cubes
    v, t = marching_cubes(torch.from_numpy(np.ascontiguousarray(vol, np.float32)).cuda(), iso)
    torch.cuda.synchronize()
    assert v.dtype == torch.float64 and t.dtype == torch.int64 and v.is_cuda and t.is_cuda
    return v.cpu().numpy(), t.cpu().numpy()


def _assert_same_mesh(vol, iso):
    v, t = _gpu_mc(vol, iso)
    vo, to = M.marching_cubes(vol, iso)
    assert v.shape == vo.shape and t.shape == to.shape
    np.testing.assert_array_equal(v.view(np.int64), vo.view(np.int64))       # bit for bit, fp64
    np.testing.assert_array_equal(t, to)
    return v, t


@pytest.mark.parametrize("case", ["smooth_37x53x29", "smooth_20", "ball", "below", "above", "ties", "cell_2x2x2",
                                  "dim1_x", "dim1_z", "dim1_all", "noise"])
def test_kernel_equals_oracle(case):
    rng = np.random.RandomState(7)
    vol, isos = {
        "smooth_37x53x29": (_smooth_field(0, (37, 53, 29)), (0.0, 0.7, -0.4)),
        "smooth_20": (_smooth_field(1, (20, 20, 20)), (0.3,)),
        "ball": (ball_field(), (0.0, 5.5)),
        "below": (rng.rand(13, 9, 11).astype(np.float32), (2.0,)),
        "above": (rng.rand(13, 9, 11).astype(np.float32), (-1.0,)),
        "ties": (tie_field(), (1.0, 0.0, 2.0)),
        "cell_2x2x2": (np.array([1, 0, 0, 0, 0, 0, 0, 1], np.float32).reshape(2, 2, 2), (0.5, 0.0)),
        "dim1_x": (rng.randn(1, 7, 9).astype(np.float32), (0.0,)),
        "dim1_z": (rng.randn(6, 7, 1).astype(np.float32), (0.0,)),
        "dim1_all": (np.ones((1, 1, 1), np.float32), (0.5,)),
        "noise": (rng.randn(23, 17, 19).astype(np.float32), (0.1, -0.2)),
    }[case]
    for iso in isos:
        v, t = _assert_same_mesh(vol, iso)
        if case in ("below", "above") or case.startswith("dim1"):
            assert v.shape == (0, 3) and t.shape == (0, 3)
        if case in ("smooth_37x53x29", "ball") or (case == "ties" and iso == 1.0):
            assert len(t) > 100 and M.closed_manifold_report(t)[0]
        if case == "ties" and iso == 2.0:                  # every value is <= 2, and a value equal to the isovalue is outside
            assert t.shape == (0, 3)


def test_rejections():
    from neuralbody_b200 import capi
    from neuralbody_b200.mcubes import marching_cubes
    lib = capi.load()
    dummy = torch.zeros(64, dtype=torch.uint8, device="cuda")
    a = capi.nb_mcubes_args()
    a.grid = a.workspace = a.counts = dummy.data_ptr()
    a.workspace_bytes = 64
    a.nx = a.ny = a.nz = 756                      # 5 * cells >= 2^31: refused on the host, nothing enqueued
    assert lib.nb_mcubes_count(ctypes.byref(a), None) == -2 and b"2^31" in lib.nb_last_error()
    a.nx = a.ny = a.nz = 8                        # a workspace too small for the grid
    assert lib.nb_mcubes_count(ctypes.byref(a), None) == -1 and b"workspace" in lib.nb_last_error()
    assert lib.nb_mcubes_workspace_bytes(8, 8, 8) > 3 * 8 * 8 * 8 * 2
    torch.cuda.synchronize()
    with pytest.raises(RuntimeError, match="CUDA"):
        marching_cubes(torch.zeros(4, 4, 4), 0.5)


def _mesh_renderer(scene):
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.networks.renderer.make_renderer import make_renderer
    net, _ = G.make_net_and_renderer(scene)
    old = cfg.renderer_module, cfg.renderer_path
    cfg.renderer_module, cfg.renderer_path = "neuralbody_b200.lib.networks.renderer.if_mesh_renderer", MESH_RENDERER
    try:
        ren = make_renderer(cfg, net)
    finally:
        cfg.renderer_module, cfg.renderer_path = old
    return net, ren


def _render(ren, batch, mesh_th):
    from neuralbody_b200.lib.config import cfg
    old = cfg.mesh_th
    cfg.mesh_th = mesh_th
    try:
        out = ren.render({k: v.cuda() for k, v in batch.items()})
    finally:
        cfg.mesh_th = old
    return out


def test_mesh_renderer_matches_reference_golden(tmp_path):
    from neuralbody_b200.mcubes import Mesh, read_ply
    gold = mesh_case.load_golden()
    scene, masks, batch = mesh_case.build_case("mesh_s03")
    assert mesh_case.case_checksum(scene, masks) == gold["input_sha256"]
    _, ren = _mesh_renderer(scene)
    assert type(ren).__module__.endswith("if_mesh_renderer")
    out = _render(ren, batch, 15.0)
    cube = out["cube"]
    assert isinstance(cube, np.ndarray) and cube.dtype == np.float64 and cube.shape == gold["cube"].shape == (72, 119, 79)
    d = np.abs(cube - gold["cube"])
    assert float(d.max()) < 2e-4, float(d.max())
    assert (cube[gold["cube"] == 0] == 0).all()                       # the scatter touches the inside points only
    mesh = out["mesh"]
    vo, to = M.marching_cubes(cube.astype(np.float32), 15.0)
    assert len(to) > 2000, len(to)                                    # thousands of triangles: not vacuous
    assert M.closed_manifold_report(to)[0]
    if isinstance(mesh, Mesh):
        np.testing.assert_array_equal(mesh.vertices.view(np.int64), vo.view(np.int64))
        np.testing.assert_array_equal(mesh.faces, to)
        # lib/visualizers/if_nerf_mesh.py:28-36: mesh.export('<result_dir>/mesh/<frame>.ply')
        path = os.path.join(str(tmp_path), "mesh", "%04d.ply" % 0)
        os.makedirs(os.path.dirname(path))
        mesh.export(path)
        v, f = read_ply(path)
        np.testing.assert_array_equal(v, mesh.vertices)
        np.testing.assert_array_equal(f, mesh.faces)
    # upstream's default mesh_th = 50 is above the synthetic body's sigma: an empty mesh, no error
    out50 = _render(ren, batch, 50)
    assert len(out50["mesh"].faces) == 0 and np.array_equal(out50["cube"], cube)


def test_mesh_render_is_deterministic():
    scene, _, batch = mesh_case.build_case("mesh_s03")
    _, ren = _mesh_renderer(scene)
    a = _render(ren, batch, 10.0)
    b = _render(ren, batch, 10.0)
    assert np.array_equal(a["cube"], b["cube"])
    assert np.array_equal(np.asarray(a["mesh"].vertices).view(np.int64), np.asarray(b["mesh"].vertices).view(np.int64))
    assert np.array_equal(np.asarray(a["mesh"].faces), np.asarray(b["mesh"].faces))


def test_full_size_mesh():
    """synth-313 at full size: the 170 x 325 x 146 grid (8.07 M points), 190 x 345 x 166 once padded."""
    scene, _, batch = mesh_case.build_case("mesh_full")
    assert tuple(batch["inside"].shape[1:]) == (170, 325, 146)
    _, ren = _mesh_renderer(scene)
    out = _render(ren, batch, 10.0)
    cube = out["cube"]
    assert cube.shape == (190, 345, 166)
    nv, nt = M.counts(cube.astype(np.float32), 10.0)
    f = np.asarray(out["mesh"].faces)
    assert (len(out["mesh"].vertices), len(f)) == (nv, nt) and nt > 10000
    assert M.closed_manifold_report(f)[0]
