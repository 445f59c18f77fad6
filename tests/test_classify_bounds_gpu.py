"""GPU: the ray classifier's cell-occupancy lookup stays inside the grid.

A sample just past the +x face of a level (floor(ix) == W) has no trilinear corner inside that level, so its features there
are exactly zero.  Its cell index must not wrap into the next bitmap row: the scene below has one non-zero voxel, on the
-x face of level LVL, placed so that such a wrapped lookup would find it occupied.  The rays run along z just past the +x
face, so every sample has all-zero features and, with skip_empty, none may be listed."""
import numpy as np
import pytest
import torch

from oracle import synth
import gpu_utils as G

pytestmark = pytest.mark.gpu

LVL = 2


def _scene():
    scene = synth.make_scene(H=16, W=16, scale=0.25, n_rays=1)
    out_sh = [int(v) for v in scene["out_sh"][0]]                  # dhw
    D, H, W = synth.level_shapes(out_sh)[LVL]
    y0, zv = H // 2 - 2, D // 2                                     # the samples' cell row; the voxel's z
    vols = [torch.zeros_like(v) for v in scene["volumes"]]
    vols[LVL][0, :, zv, y0 + 2, 0] = 1.0       # occupies cells (0..1, y0+2..y0+3, zv..zv+1), the wrap target of (W+1, y0+1, *)
    scene["volumes"] = vols

    # canonical (SMPL-frame) point of level-LVL grid index (ix, iy, iz): the inverse of world_to_grid's normalisation
    bmin = scene["bounds"][0, 0].double().numpy()                  # xyz
    vox = np.asarray(scene["voxel_size"], np.float64)[::-1]        # xyz
    sh = np.asarray(out_sh, np.float64)[::-1]                      # xyz
    size = np.asarray([W, H, D], np.float64)
    canon = lambda i: bmin + vox * sh * np.asarray(i, np.float64) / (size - 1)
    R = scene["R"][0].double().numpy()
    Th = scene["Th"].reshape(-1, 3)[0].double().numpy()
    c0, c1 = canon([W + 0.5, y0 + 0.5, 1.0]), canon([W + 0.5, y0 + 0.5, D - 2.0])
    o = c0 @ R.T + Th                                              # world = canonical R^T + Th
    d = (c1 - c0) @ R.T
    dist = float(np.linalg.norm(d))
    scene["ray_o"] = torch.tensor(o, dtype=torch.float32).reshape(1, 1, 3)
    scene["ray_d"] = torch.tensor(d / dist, dtype=torch.float32).reshape(1, 1, 3)
    scene["near"] = torch.zeros(1, 1)
    scene["far"] = torch.full((1, 1), dist, dtype=torch.float32)
    return scene


def test_samples_past_the_grid_face_are_not_listed():
    scene = _scene()
    net, ren = G.make_net_and_renderer(scene)
    ren.stats = torch.zeros(8, dtype=torch.int64, device="cuda")
    dense = G.render_product(scene, precision="tc_fp16x3", want_raw=True, renderer=ren, net=net, skip_empty=False)
    assert int(ren.stats[1]) == 64                                 # the ray's 64 samples, all listed
    ren.stats.zero_()
    sparse = G.render_product(scene, precision="tc_fp16x3", want_raw=True, renderer=ren, net=net, skip_empty=True)
    assert int(ren.stats[1]) == 0                                  # all-zero features: nothing is listed
    raw = sparse["raw"].reshape(-1, 4)
    assert float(raw[:, :3].abs().max()) == 0.0                    # the constant skipped-sample record (0, 0, 0, sigma)
    assert float(raw[:, 3].max()) < 0.0 and torch.equal(raw[:, 3], raw[:1, 3].expand(raw.shape[0]))
    for k in ("rgb_map", "depth_map", "acc_map", "weights", "disp_map"):
        assert torch.equal(torch.nan_to_num(dense[k], nan=-1.0), torch.nan_to_num(sparse[k], nan=-1.0)), k
