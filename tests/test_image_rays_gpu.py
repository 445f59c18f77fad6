"""nb_image_rays / nb_image_rays_f64: the demo datasets' render_utils.image_rays on the GPU, bit for bit, and the renderers
rendering from the camera batch exactly as from upstream's rays."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from conftest import ROOT
from tools import demo_case as DC

pytestmark = pytest.mark.gpu

KEYS = ("ray_o", "ray_d", "near", "far", "mask_at_box")


def device_rays(RT, K, bounds, H, W):
    from neuralbody_b200 import rays
    out = rays.camera_image_rays(RT, K, bounds, H, W)
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in out]


def assert_same(got, want, label):
    for k, g, w in zip(KEYS, got, want):
        w = np.asarray(w)
        assert g.shape == w.shape, "%s %s shape %s != %s" % (label, k, g.shape, w.shape)
        if k == "mask_at_box":
            assert np.array_equal(g, w), "%s mask_at_box: %d pixels differ" % (label, int((g != w).sum()))
        else:
            assert np.array_equal(g.view(np.uint32), np.asarray(w, np.float32).view(np.uint32)), \
                "%s %s: %d values differ" % (label, k, int((g != w).sum()))


@pytest.mark.parametrize("golden", [DC.GOLDEN_MV, DC.GOLDEN_MONO], ids=["float64_multi_view", "float32_monocular"])
def test_goldens_bit_for_bit(golden):
    g = DC.load_golden(golden)
    for v, c in g["views"].items():
        got = device_rays(c["RT"], c["K"], c["bounds"], g["H"], g["W"])
        assert_same(got, [c[k] for k in KEYS], "%s view %d" % (os.path.basename(golden), v))
        assert len(got[2]) == int(c["mask_at_box"].sum()) > 0


def _orbit():
    z = np.load(DC.ORBIT)
    for j, v in enumerate(z["mv_views"]):
        yield "gen_path view %d" % v, z["mv_RT"][j], z["mv_K"], z["mv_bounds"], tuple(z["mv_HW"])
    for j, v in enumerate(z["mono_views"]):
        yield "monocular angle %d" % v, z["mono_RT"], z["mono_K"], z["mono_bounds"][j], tuple(z["mono_HW"])


def test_full_size_orbits_match_the_restatement():
    """512 x 512 views of the 144-view gen_path orbit (float64 camera) and 540 x 540 views of the People-Snapshot orbit
    (float32 camera) against the numpy restatement: 0 differing rays."""
    for label, RT, K, b, (H, W) in _orbit():
        got = device_rays(RT, K, b, H, W)
        want = DC.image_rays_numpy(RT, K, b, H, W)
        n_diff = int((got[4] != want[4]).sum())
        print("%s: %d rays, %d mask_at_box flips" % (label, int(want[4].sum()), n_diff))
        assert_same(got, want, label)


def _look_at(c, target):
    z = (target - c) / np.linalg.norm(target - c)
    x = np.cross(np.array([0., 1., 0.]), z); x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z])
    RT = np.eye(4); RT[:3, :3] = R; RT[:3, 3] = -R @ c
    return RT


BOX = np.array([[-0.3, -0.9, -0.2], [0.3, 0.8, 0.25]], np.float32)
K64 = np.array([[300., 0, 40.5], [0, 301., 30.5], [0, 0, 1.]])


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_view_that_misses_the_box(dtype):
    """get_near_far tests the whole line (near may be negative), so the lines themselves must pass the box: a camera beside
    it, looking past it."""
    RT = _look_at(np.array([2., 0., -3.]), np.array([2., 0., 3.]))[:3].astype(dtype)
    assert not DC.image_rays_numpy(RT, K64.astype(dtype), BOX, 60, 80)[4].any()
    got = device_rays(RT, K64.astype(dtype), BOX, 60, 80)
    assert len(got[0]) == len(got[2]) == len(got[3]) == 0 and got[0].shape == (0, 3)
    assert got[4].shape == (4800,) and not got[4].any()


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_camera_inside_the_box(dtype):
    RT = _look_at(np.array([0.05, 0.1, 0.0]), np.array([0.3, 0.2, 2.]))[:3].astype(dtype)
    want = DC.image_rays_numpy(RT, K64.astype(dtype), BOX, 60, 80)
    assert want[4].all() and (want[2] < 0).all()       # every ray starts inside: near is behind the camera
    assert_same(device_rays(RT, K64.astype(dtype), BOX, 60, 80), want, "inside")


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_axis_parallel_rays_take_the_clamp(dtype):
    """R = I, T = 0 and the principal point on a pixel centre with a power-of-two focal length (inv(K) exact in both
    dtypes): that pixel's column and row have ray_d x or y exactly 0, so the 1e-5 / -1e-5 viewdir clamp decides their
    slabs."""
    RT = np.eye(4)[:3].astype(dtype)
    K = np.array([[256., 0, 40.], [0, 256., 30.], [0, 0, 1.]], dtype)
    box = BOX + np.array([0., 0., 3.], np.float32)
    want = DC.image_rays_numpy(RT, K, box, 60, 80)
    zero = (want[1][:, 0] == 0) | (want[1][:, 1] == 0)
    assert zero.sum() > 10
    assert_same(device_rays(RT, K, box, 60, 80), want, "axis-parallel")


# ----------------------------------------------------------------------------- renderers
def _scene_and_cameras():
    from tools import mesh_mono_case as MM
    scene = MM.make_scene(0.3)
    H, W = 100, 75
    pkl = MM.camera_pkl(scene, H, W)
    K64 = MM.get_camera(pkl)["K"]
    msk = (MM.silhouette(scene, K64, H, W, 2) != 0).astype(np.uint8)
    return scene, K64, msk, H, W


def _render(mod, batch, precision, H, W):
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.networks.make_network import load_source
    from gpu_utils import make_net_and_renderer
    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.raw_noise_std = 64, 0.0, False, 0
    cfg.render_precision, cfg.render_volume_dtype, cfg.chunk, cfg.render_skip_empty = precision, "auto", 0, True
    net, _ = make_net_and_renderer(batch.pop("_scene"))
    net.train(False)
    path = os.path.join(ROOT, "neuralbody_b200", "lib", "networks", "renderer", mod + ".py")
    ren = load_source("neuralbody_b200.lib.networks.renderer." + mod, path).Renderer(net)
    cfg.H, cfg.W, cfg.ratio = H, W, 1.0
    with torch.no_grad():
        out = ren.render(batch)
    torch.cuda.synchronize()
    return {k: v.detach().cpu() for k, v in out.items()}


@pytest.mark.parametrize("precision", ["fp32", "tc_fp16x3"])
@pytest.mark.parametrize("kind", ["mmsk_demo", "mmsk_perform", "msk_mono"])
def test_render_from_camera_equals_render_from_rays(kind, precision):
    scene, K, msk, H, W = _scene_and_cameras()
    dev = "cuda:0"
    cb = scene["can_bounds"][0].numpy()
    if kind == "msk_mono":      # float32 camera, one snapshot mask (monocular_demo_dataset)
        RT = np.concatenate([np.eye(3), np.zeros((3, 1))], axis=1).astype(np.float32)
        Kc = K.astype(np.float32)
        mod = "if_nerf_renderer_msk"
        extra = {"msk": torch.from_numpy(msk)[None], "RT": torch.from_numpy(RT)[None], "K": torch.from_numpy(Kc)[None],
                 "R0_snap": scene["R"], "Th0_snap": scene["Th"]}
    else:                       # float64 camera (a gen_path render_w2c is (4,4)), mask views from a float32 copy
        RT = np.eye(4) if kind == "mmsk_demo" else np.eye(4)[:3].copy()
        RT[:3, 3] = (0.004, -0.002, 0.01)
        Kc = K
        mod = "if_nerf_renderer_mmsk"
        extra = {"msks": torch.from_numpy(msk)[None, None], "RT": torch.from_numpy(RT[:3].astype(np.float32))[None, None],
                 "Ks": torch.from_numpy(K.astype(np.float32))[None, None]}
    ray_o, ray_d, near, far, mask = DC.image_rays_numpy(RT, Kc, cb, H, W)
    base = {k: scene[k] for k in ("coord", "out_sh", "bounds", "R", "Th", "latent_index")}
    base.update(extra)
    rays_batch = {k: v.to(dev) for k, v in base.items()}
    rays_batch.update({"ray_o": torch.from_numpy(ray_o)[None].to(dev), "ray_d": torch.from_numpy(ray_d)[None].to(dev),
                       "near": torch.from_numpy(near)[None].to(dev), "far": torch.from_numpy(far)[None].to(dev)})
    cam_batch = {k: v.to(dev) for k, v in base.items()}
    cam_batch.update({"cam_RT": torch.from_numpy(RT)[None].to(dev), "cam_K": torch.from_numpy(Kc)[None].to(dev),
                      "can_bounds": torch.from_numpy(cb)[None].to(dev)})
    want = _render(mod, dict(rays_batch, _scene=scene), precision, H, W)
    # the renderer sets batch['mask_at_box'] on the camera batch it was handed
    cam_batch["_scene"] = scene
    got = _render(mod, cam_batch, precision, H, W)
    assert cam_batch["mask_at_box"].shape == (1, H * W) and cam_batch["mask_at_box"].device.type == "cuda"
    assert np.array_equal(cam_batch["mask_at_box"][0].cpu().numpy(), mask)
    assert 0 < int(mask.sum()) < H * W
    for k in want:
        a, b = got[k].numpy(), want[k].numpy()
        assert a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32)), "%s %s differs" % (kind, k)


def test_mixed_camera_raises():
    from neuralbody_b200 import rays
    with pytest.raises(ValueError):
        rays.camera_image_rays(np.eye(4), K64.astype(np.float32), BOX, 8, 8)


def test_camera_from_meta_on_the_host_equals_camera_on_the_device():
    """The drop-ins' host copy of the camera in batch['meta'] (which upstream's visualize loop leaves on the host) gives the
    rays and mask_at_box of the same camera read from the device tensors."""
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.networks.renderer.if_nerf_renderer import Renderer
    z = np.load(DC.ORBIT)
    cfg.H, cfg.W, cfg.ratio = 1024, 1024, 0.5
    cam = {"cam_RT": torch.from_numpy(z["mv_RT"][1])[None], "cam_K": torch.from_numpy(z["mv_K"])[None],
           "can_bounds": torch.from_numpy(z["mv_bounds"])[None]}
    coord = torch.zeros((1, 1, 3), dtype=torch.int32, device="cuda:0")
    on_dev = dict({k: v.cuda() for k, v in cam.items()}, coord=coord)
    on_host = dict(on_dev, meta=cam)
    ren = Renderer.__new__(Renderer)
    a, b = ren.camera_rays(on_dev), ren.camera_rays(on_host)
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))
    assert torch.equal(on_dev["mask_at_box"], on_host["mask_at_box"]) and int(on_host["mask_at_box"].sum()) == a[0].shape[1]
    want = DC.image_rays_numpy(z["mv_RT"][1], z["mv_K"], z["mv_bounds"], 512, 512)
    assert np.array_equal(b[2][0].cpu().numpy(), want[2])
