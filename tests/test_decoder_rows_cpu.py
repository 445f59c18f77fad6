"""CPU: the tile builder of tests/test_decoder_rows_gpu.py (oracle/decoder_tiles.py) builds what it claims, and the row
emulation of the decoder (oracle/tc_decoder_model.py) agrees with the float64 oracle and restates the kernel's roundings."""
import torch

from oracle import decoder_tiles as T
from oracle import neuralbody_oracle as O
from oracle import tc_decoder_model as M


def test_limit_half_tiles_hit_their_distinct_voxel_targets():
    for level, (first, second) in ((3, (64, 65)), (2, (64, 65)), (1, (128, 129)), (0, (128, 129))):
        g = T.limit_group(level, first, second)
        assert g.shape == (128, 3)
        assert bool((T.classes(g) == level).all()), level
        assert T.distinct_voxels(g[:64], level) == first
        assert T.distinct_voxels(g[64:], level) == second


def test_regions_give_their_classes_and_level_gaps():
    for region, cls in ((3, 3), (2, 2), (1, 1), ("gap", 1), (0, 0), ("empty", -1)):
        q = T.random_points(region, 256, seed=3)
        assert bool((T.classes(q) == cls).all()), region
    gap = T.random_points("gap", 64, seed=4)
    assert bool(T.occupied(gap, 3).all() and T.occupied(gap, 1).all())
    assert not bool(T.occupied(gap, 2).any() or T.occupied(gap, 0).any())
    assert bool((T.classes(T.random_points("empty", 8, seed=5), skip=False) == 3).all())


def test_boundary_points_straddle_every_level():
    b = T.boundary_points()
    for l in range(4):
        size = T.level_size(l)
        f = torch.floor(b / (1 << l)).long()
        low = (f == -1).any(1)
        high = torch.stack([f[:, a] == size[a] - 1 for a in range(3)], 1).any(1)
        assert bool((low | high).all()), l
    assert set(T.classes(b).tolist()) == {0, 1, 3}


def test_tile_stats_of_the_limit_groups():
    gs = [T.limit_group(3, 64, 65), T.limit_group(2, 64, 65), T.limit_group(1, 128, 129), T.limit_group(0, 128, 129)]
    st = T.tile_stats(gs)
    assert st[0] == 4 and st[1] == 512 and st[4] == 8 + 16 + 20 + 22
    # one half direct on level 3 (65 > 64), one on level 2; the level-1 and level-0 129 halves are direct
    assert st[6] == 2 and st[7] == 2 and st[5] == 2 + 4 + 4 + 4 - 2


def test_world_points_land_on_their_grid_coordinates():
    R, Th, bounds = T.frame(1)
    q0 = torch.cat([T.random_points(0, 64, 1), T.random_points(3, 64, 2), T.boundary_points()])
    w = T.world_points(q0, R, Th, bounds)
    g = M.world_to_grid_f32(w, R, Th, bounds, T.VOXEL, T.OUT_SH)
    ix = ((g.double() + 1) * 0.5) * torch.tensor([n - 1 for n in T.N0], dtype=torch.float64)
    assert float((ix - q0).abs().max()) < 1e-3


def test_kernel_gather_restatement_matches_grid_sample():
    R, Th, bounds = T.frame(2)
    vols = T.make_volumes(7)
    q0 = torch.cat([T.random_points(r, 64, 8) for r in (3, 2, 1, 0, "gap")] + [T.boundary_points()])
    w = T.world_points(q0, R, Th, bounds)
    got = M.gather_f32(M.world_to_grid_f32(w, R, Th, bounds, T.VOXEL, T.OUT_SH), [v[0] for v in vols])
    sp = {"R": R[None].double(), "Th": Th[None].double(), "bounds": bounds[None].double(), "out_sh": list(T.OUT_SH)}
    grid = O.get_grid_coords(O.pts_to_can_pts(w[None].double(), sp["R"], sp["Th"]), sp["bounds"], sp["out_sh"], T.VOXEL)
    want = O.interpolate_features(grid, [v.double() for v in vols])[0].t()
    # the float32 world -> grid chain places a point within ~1e-5 voxel of the float64 one (up to 193 voxels per axis)
    assert float((got.double() - want).abs().max()) < 1e-4
    assert float(want.abs().sum()) > 0


def test_roundings():
    x = torch.tensor([1.0 + 2 ** -12, -3.0 - 2 ** -11 - 2 ** -20, 2 ** -16 * 1.75 + 2 ** -30, 65504.0, 0.0])
    hi, lo = M.split_act(x)
    assert torch.equal(hi, torch.tensor([1.0, -3.0, 2 ** -16 * 1.75, 65504.0, 0.0]))
    assert float(lo[0]) == 2 ** -12
    # below fp16's smallest normal the truncation runs on the 2^-24 grid, and lo only carries x - trunc13(x)
    y = torch.tensor([2 ** -20 * 1.3])
    assert float(M.f16_rz(y)) == float(torch.floor(y.double() * 2 ** 24) * 2 ** -24)
    assert torch.equal(M.fma32(torch.tensor([3.0]), torch.tensor([1.0 / 3]), torch.tensor([-1.0])),
                       torch.tensor([float(torch.tensor(3.0, dtype=torch.float64) * float(torch.tensor(1.0 / 3)) - 1.0)]))


def test_probes_meet_staged_and_direct_half_tiles():
    """The probe contexts of test_decoder_rows_gpu.py: beside local neighbours every gathered level of the probes' half tile
    is staged, beside random class-0 points every one is direct."""
    p = T.probe_points()
    assert bool((T.classes(p) == 0).all())
    head = torch.cat([p, T.local_points(0, 112, seed=21)])
    tail = torch.cat([T.random_points(0, 112, seed=22), p])
    assert T.half_paths(head[:64]) == ["staged"] * 4
    assert T.half_paths(tail[64:]) == ["direct"] * 4


def test_render_rays_reproduce_the_groups():
    """Sample 1 of a designed ray is its sample 0 moved by one level-3 voxel along y: same classes, same distinct voxels."""
    R, Th, bounds = T.frame(0)
    groups = [T.limit_group(3, 64, 65), T.random_points(0, 128, 1, ymax=40), T.random_points(2, 128, 2, ymax=40),
              T.random_points("gap", 128, 3, ymax=40)]
    o, d, z, q = T.render_rays(groups, R, Th, bounds)
    for s in range(2):
        w = M.sample_points_f32(o, d, z)[:, s]
        g = M.world_to_grid_f32(w, R, Th, bounds, T.VOXEL, T.OUT_SH)
        ix = ((g.double() + 1) * 0.5) * torch.tensor([n - 1 for n in T.N0], dtype=torch.float64)
        assert float((ix - q[:, s]).abs().max()) < 1e-3
    moved = T.render_groups(groups)[4:]
    for a, b in zip(groups, moved):
        assert torch.equal(T.classes(a), T.classes(b))
        for l in range(4):
            assert T.distinct_voxels(a[:64], l) == T.distinct_voxels(b[:64], l)
