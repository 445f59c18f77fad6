"""CPU: the marching-cubes table and its numpy restatement (oracle/mcubes_oracle.py), the mesh renderer's cube against the
golden made by the unmodified reference (tests/golden/mesh_s03.npz), the grid / `inside` restatement, the PLY writer, and
the mesh entry points' host-side checks."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch
from scipy import ndimage

from conftest import ROOT
from oracle import mcubes_oracle as M
from oracle import mesh_case
from tools import gen_mc_table

NB_ERR_BAD_ARG, NB_ERR_UNSUPPORTED = -1, -2     # include/neuralbody_b200.h


def test_generator_reproduces_committed_header():
    with open(os.path.join(ROOT, "neuralbody_b200", "csrc", "nb_mc_table.h")) as f:
        assert f.read() == gen_mc_table.render_header()


def test_every_case_closes_into_loops_of_at_most_five_triangles():
    table = gen_mc_table.build_table()
    hist = [0] * 6
    for case, tris in enumerate(table):
        loops = gen_mc_table.case_loops(case)          # asserts one in / one out segment per crossed edge
        crossed = sorted(e for loop in loops for e in loop)
        inside = [(case >> v) & 1 for v in range(8)]
        want = sorted(gen_mc_table.edge_of(c0, c0 | (1 << a)) for c0 in range(8) for a in range(3)
                      if not (c0 >> a) & 1 and inside[c0] != inside[c0 | (1 << a)])
        assert crossed == want, case
        assert max((len(l) for l in loops), default=0) <= 7
        assert len(tris) == sum(len(l) - 2 for l in loops) <= 5
        # within the case, every triangle edge is used once in each direction or lies on the boundary loop
        d = {}
        for a, b, c in tris:
            for e in ((a, b), (b, c), (c, a)):
                d[e] = d.get(e, 0) + 1
        assert all(n == 1 for n in d.values()), case
        hist[len(tris)] += 1
    assert hist == [2, 16, 50, 80, 76, 32]
    assert table[0] == [] and table[255] == []


def _check_mesh(vol, iso, verts, tris):
    assert np.isfinite(verts).all()
    ok, msg = M.closed_manifold_report(tris)
    assert ok, msg
    if len(tris):
        assert tris.min() >= 0 and tris.max() < len(verts)
        assert len(np.unique(tris)) == len(verts)                 # every vertex is used
    v64 = vol.astype(np.float64)
    fl = np.floor(verts).astype(np.int64)
    frac = verts - fl
    nonint = (frac != 0).sum(1)
    assert (nonint <= 1).all()                                     # on a grid edge
    on_pt = nonint == 0
    assert (v64[fl[on_pt, 0], fl[on_pt, 1], fl[on_pt, 2]] == iso).all()   # t = 0 or 1 only on a tie
    e = ~on_pt
    ax = np.argmax(frac[e] != 0, axis=1)
    p = fl[e]
    q = p.copy()
    q[np.arange(len(q)), ax] += 1
    f0, f1 = v64[p[:, 0], p[:, 1], p[:, 2]], v64[q[:, 0], q[:, 1], q[:, 2]]
    assert ((f0 > iso) != (f1 > iso)).all()                        # a crossed edge
    interp = f0 + frac[e][np.arange(len(ax)), ax] * (f1 - f0)
    np.testing.assert_allclose(interp, iso, rtol=0, atol=1e-9 * max(1.0, float(np.abs(v64).max())))


def _smooth_field(seed, shape, sigma=2.0):
    rng = np.random.RandomState(seed)
    f = ndimage.gaussian_filter(rng.randn(*shape), sigma)
    f = (f / f.std()).astype(np.float32)
    for a in range(3):                                             # keep the surface off the grid boundary
        idx = [slice(None)] * 3
        for s in (0, -1):
            idx[a] = s
            f[tuple(idx)] = -10.0
    return f


def ball_field(n=48, r=20.0, c=(23.3, 24.1, 22.7)):
    g = np.stack(np.meshgrid(*[np.arange(n, dtype=np.float64)] * 3, indexing="ij"), -1)
    return (r - np.linalg.norm(g - np.asarray(c), axis=-1)).astype(np.float32)


def tie_field(seed=3, shape=(17, 13, 19)):
    rng = np.random.RandomState(seed)
    f = rng.randint(0, 3, size=shape).astype(np.float32)          # values 0, 1, 2 at isovalue 1: many exact ties
    f[[0, -1]] = 0
    f[:, [0, -1]] = 0
    f[:, :, [0, -1]] = 0
    return f


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_oracle_mesh_on_smooth_random_fields(seed):
    shape = [(37, 53, 29), (20, 20, 20), (31, 17, 45), (12, 40, 25)][seed]
    f = _smooth_field(seed, shape)
    for iso in (0.0, 0.7, -0.4):
        verts, tris = M.marching_cubes(f, iso)
        assert len(tris) > 50
        _check_mesh(f, iso, verts, tris)
        assert M.signed_volume(verts, tris) > 0
        assert M.counts(f, iso) == (len(verts), len(tris))


def test_oracle_mesh_on_white_noise_is_closed():
    """Every ambiguous face configuration shows up here; the table still gives a closed manifold."""
    rng = np.random.RandomState(11)
    for _ in range(20):
        f = rng.randn(10, 9, 11).astype(np.float32)
        f[[0, -1]] = f[:, [0, -1]] = f[:, :, [0, -1]] = -5
        verts, tris = M.marching_cubes(f, 0.1)
        _check_mesh(f, 0.1, verts, tris)


def test_oracle_ball_volume():
    f = ball_field()
    verts, tris = M.marching_cubes(f, 0.0)
    _check_mesh(f, 0.0, verts, tris)
    vol = M.signed_volume(verts, tris)
    want = 4.0 / 3.0 * math.pi * 20.0 ** 3
    assert vol > 0 and abs(vol / want - 1) < 0.01, vol / want


def test_oracle_ties_count_as_outside():
    f = tie_field()
    verts, tris = M.marching_cubes(f, 1.0)
    assert len(tris) > 100
    _check_mesh(f, 1.0, verts, tris)
    # a value equal to the isovalue is outside: the mesh of `f` at 1 has the topology of (f == 2) at 0.5, with each vertex
    # on the same grid edge (at its end instead of its midpoint)
    v2, t2 = M.marching_cubes((f == 2).astype(np.float32), 0.5)
    np.testing.assert_array_equal(tris, t2)
    assert np.abs(verts - v2).max() == 0.5 and ((verts - v2 != 0).sum(1) <= 1).all()


def test_oracle_degenerate_grids():
    for shape in ((1, 5, 5), (5, 1, 5), (4, 4, 1), (1, 1, 1)):
        v, t = M.marching_cubes(np.random.RandomState(0).randn(*shape).astype(np.float32), 0.0)
        assert v.shape == (0, 3) and t.shape == (0, 3)
    f = np.zeros((2, 2, 2), np.float32)
    f[0, 0, 0] = 1
    v, t = M.marching_cubes(f, 0.5)
    assert v.shape == (3, 3) and t.shape == (1, 3)
    np.testing.assert_array_equal(np.sort(v, 0), np.sort(np.array([[0.5, 0, 0], [0, 0.5, 0], [0, 0, 0.5]]), 0))
    n = np.cross(v[t[0, 1]] - v[t[0, 0]], v[t[0, 2]] - v[t[0, 0]])
    assert (n > 0).all()                                            # points away from the inside corner (0,0,0)


def test_oracle_cube_matches_reference_golden():
    """calculate_density of the oracle on the inside points, scattered and padded as if_mesh_renderer.py:40-47 does, equals
    the cube the unmodified reference handed to mcubes.marching_cubes."""
    from oracle import neuralbody_oracle as O
    gold = mesh_case.load_golden()
    scene, masks, batch = mesh_case.build_case("mesh_s03")
    assert mesh_case.case_checksum(scene, masks) == gold["input_sha256"]
    inside = batch["inside"][0].numpy()
    wpts = batch["pts"][0][inside.astype(bool)][None]
    with torch.no_grad():
        alpha = O.calculate_density(scene["weights"], wpts, scene["volumes"], O.prepare_sp_input(scene), scene["voxel_size"])
    cube = M.pad_cube(inside, alpha[0, :, 0].numpy())
    assert cube.dtype == np.float64 and cube.shape == tuple(s + 20 for s in gold["shape"]) == (72, 119, 79)
    np.testing.assert_array_equal(cube, gold["cube"])
    # the synthetic body's sigma stays below upstream's default mesh_th = 50; the mesh tests use isovalues inside its range
    assert -20 < cube.min() < -5 and 20 < cube.max() < 50


def test_grid_and_inside_restatement_match_reference():
    import hashlib
    gold = mesh_case.load_golden()
    _, _, batch = mesh_case.build_case("mesh_s03")
    pts, inside = batch["pts"][0].numpy(), batch["inside"][0].numpy()
    assert pts.shape == gold["shape"] + (3,) and pts.dtype == np.float32
    assert hashlib.sha256(np.ascontiguousarray(pts).tobytes()).hexdigest() == gold["pts_sha256"]
    np.testing.assert_array_equal(inside, gold["inside"])
    assert 0.05 < inside.mean() < 0.5


def test_mesh_ply_roundtrip(tmp_path):
    from neuralbody_b200.mcubes import Mesh, read_ply
    verts, tris = M.marching_cubes(ball_field(n=24, r=8.0, c=(11.5, 12.2, 11.8)), 0.0)
    mesh = Mesh(verts, tris)
    path = str(tmp_path / "0000.ply")
    mesh.export(path)
    v, f = read_ply(path)
    np.testing.assert_array_equal(v, verts)
    np.testing.assert_array_equal(f, tris)
    assert v.dtype == np.float64 and f.dtype == np.int64
    empty = str(tmp_path / "empty.ply")
    Mesh(np.zeros((0, 3)), np.zeros((0, 3), np.int64)).export(empty)
    v, f = read_ply(empty)
    assert v.shape == (0, 3) and f.shape == (0, 3)


def test_mesh_entry_points_check_arguments_on_the_host(built_lib):
    from neuralbody_b200 import capi
    lib = capi.load()
    a = capi.nb_mcubes_args()
    assert lib.nb_mcubes_count(ctypes.byref(a), None) == NB_ERR_BAD_ARG and b"null" in lib.nb_last_error()
    a.grid = a.workspace = a.counts = 256                 # never dereferenced: every check below happens first
    a.nx, a.ny, a.nz = 0, 4, 4
    assert lib.nb_mcubes_count(ctypes.byref(a), None) == NB_ERR_BAD_ARG
    # 5 * cells >= 2^31 (32-bit offsets): refused before anything is launched, no allocation involved
    a.nx, a.ny, a.nz = 756, 756, 756
    assert 5 * 755 ** 3 >= 2 ** 31 > 5 * 754 ** 3
    assert lib.nb_mcubes_count(ctypes.byref(a), None) == NB_ERR_UNSUPPORTED and b"2^31" in lib.nb_last_error()
    assert lib.nb_mcubes_emit(ctypes.byref(a), None) == NB_ERR_UNSUPPORTED
    a.nx, a.ny, a.nz = 755, 755, 755                      # within the limit: fails later (workspace, or no device here)
    assert lib.nb_mcubes_count(ctypes.byref(a), None) not in (0, NB_ERR_UNSUPPORTED)
    a.nx, a.ny, a.nz = 2, 2, 400000000                    # few cells, but 3 * points >= 2^31
    assert lib.nb_mcubes_count(ctypes.byref(a), None) == NB_ERR_UNSUPPORTED
    assert lib.nb_mcubes_workspace_bytes(0, 3, 3) == 0
    from neuralbody_b200.mcubes import marching_cubes
    with pytest.raises(RuntimeError, match="CUDA"):
        marching_cubes(torch.zeros(4, 4, 4), 0.5)


def test_mesh_renderer_contract_without_gpu(built_lib):
    """Selected by path like every renderer; refuses a batch without the grid keys, and CPU tensors."""
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.config.config import _defaults
    from neuralbody_b200.lib.networks import make_network
    from neuralbody_b200.lib.networks.make_network import load_source
    assert _defaults().mesh_th == 50
    path = os.path.join(ROOT, "neuralbody_b200", "lib", "networks", "renderer", "if_mesh_renderer.py")
    mod = load_source("neuralbody_b200.lib.networks.renderer.if_mesh_renderer", path)
    cfg.num_train_frame = 60
    ren = mod.Renderer(make_network(cfg))
    with pytest.raises(KeyError, match="inside"):
        ren.render({"pts": torch.zeros(1, 2, 2, 2, 3)})
    with pytest.raises(KeyError, match="pts"):
        ren.render({"inside": torch.zeros(1, 2, 2, 2)})
    with pytest.raises(RuntimeError, match="CUDA"):
        ren.render({"pts": torch.zeros(1, 2, 2, 2, 3), "inside": torch.zeros(1, 2, 2, 2, dtype=torch.uint8)})
