"""nb_vis_frame and the visualizer drop-ins on the GPU: the goldens made by the unmodified reference visualizers, the
numpy restatement (oracle/vis_frames.py, pinned to the reference by test_vis_frames_cpu) on random views, the errors,
visualize() without host synchronisation, Renderer.render -> Visualizer.visualize end to end for both modules, and the
rotate-SMPL drop-in's item against upstream's rays."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import vis_frames as O
from tools import vis_case as VC

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


@pytest.fixture(autouse=True)
def _restore_cfg():
    from neuralbody_b200.lib.config import cfg
    saved = cfg.clone()
    yield
    cfg.clear()
    cfg.update(saved)


def _gpu(rgb, mask, H, W, white=0):
    from neuralbody_b200 import vis_frame
    v = vis_frame.vis_frame(torch.from_numpy(rgb).to(DEV), torch.from_numpy(mask).to(DEV), H, W, white)
    torch.cuda.synchronize()
    return vis_frame.parse(v.result.cpu().numpy()), v.frame.cpu().numpy()


@pytest.mark.parametrize("name", sorted(VC.CASES))
def test_goldens(name):
    want = VC.load_golden()[name]
    rgb, mask, (H, W, white) = VC.case(name)
    assert VC.checksum(rgb, mask) == bytes(want["sha256"]).decode()
    (status, count), frame = _gpu(rgb, mask, H, W, white)
    assert status == 0 and count == rgb.shape[0]
    assert np.array_equal(frame, want["frame"]), (name, int((frame != want["frame"]).sum()))


RANDOM = [(1, 1, 0, 1), (3, 5, 1, 2), (37, 41, 0, 3), (512, 512, 1, 4), (1080, 1920, 0, 5), (1080, 1920, 1, 6),
          (1001, 999, 0, 7)]


@pytest.mark.parametrize("case", RANDOM, ids=["%dx%d_w%d" % c[:3] for c in RANDOM])
def test_random_views_equal_the_restatement(case):
    H, W, white, seed = case
    rgb, mask = VC.random_view(H, W, seed)
    (status, count), frame = _gpu(rgb, mask, H, W, white)
    assert status == 0 and count == rgb.shape[0]
    assert np.array_equal(frame, O.frame(rgb, mask, H, W, white))


def test_one_ray_broadcasts_and_counts_mismatch():
    from neuralbody_b200 import capi
    rgb, mask, (H, W, white) = VC.case("white")
    (status, _), frame = _gpu(rgb[:1], mask, H, W, white)
    assert status == capi.NB_VIS_OK and np.array_equal(frame, O.frame(rgb[:1], mask, H, W, white))
    for bad in (rgb[:-1], rgb[:0], np.concatenate([rgb, rgb[:2]])):
        (status, count), _ = _gpu(np.ascontiguousarray(bad), mask, H, W, white)
        assert status == capi.NB_VIS_COUNT and count == rgb.shape[0]


# ----------------------------------------------------------------------------- the drop-ins
def _cfg(H, W, white, exp_name="vis"):
    from neuralbody_b200.lib.config import cfg
    cfg.H, cfg.W, cfg.ratio, cfg.white_bkgd, cfg.exp_name = H, W, 1.0, bool(white), exp_name
    return cfg


def _visualizer(kind):
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.networks.make_network import load_source
    path = cfg.visualizer_path.replace("if_nerf_demo", "if_nerf_" + kind)
    return load_source(cfg.visualizer_module.replace("if_nerf_demo", "if_nerf_" + kind), path).Visualizer()


def _png_bytes(frame, path):
    import cv2
    assert cv2.imwrite(str(path), frame)
    return open(str(path), "rb").read()


def _view(rgb, mask, fi, vi, device=DEV):
    return ({"rgb_map": torch.from_numpy(rgb)[None].to(device)},
            {"mask_at_box": torch.from_numpy(mask)[None].to(device), "frame_index": torch.tensor([fi]).to(device),
             "view_index": torch.tensor([vi]).to(device)})


def test_errors_are_raised_at_the_next_call(monkeypatch, tmp_path):
    pytest.importorskip("cv2")
    monkeypatch.chdir(tmp_path)
    rgb, mask, (H, W, white) = VC.case("white")
    _cfg(H, W, white)
    vis = _visualizer("demo")
    with pytest.raises(ValueError, match="cannot reshape"):     # at once
        vis.visualize(*_view(rgb, mask[:-1], 0, 0))
    vis.visualize(*_view(rgb[:-1], mask, 0, 1))                 # queued: the count is checked on the writer
    with pytest.raises(ValueError, match="shape mismatch"):
        vis.flush()
    vis.visualize(*_view(rgb[:-2], mask, 0, 2))
    torch.cuda.synchronize()
    vis._writer._q.join()
    with pytest.raises(ValueError, match="shape mismatch"):
        vis.visualize(*_view(rgb, mask, 0, 3))
    vis.visualize(*_view(rgb, mask, 0, 4))
    vis.flush()
    assert sorted(os.listdir(tmp_path / "data" / "render" / "vis" / "frame_0000")) == ["0004.png"]


def test_visualize_does_not_synchronise(monkeypatch, tmp_path):
    """Under torch's sync debug mode "error", visualize() with device indices and with host indices runs to the end."""
    cv2 = pytest.importorskip("cv2")
    monkeypatch.chdir(tmp_path)
    rgb, mask = VC.random_view(540, 540, 11)
    _cfg(540, 540, 0)
    vis = _visualizer("perform")
    views = [_view(rgb, mask, 7, 0), _view(rgb, mask, 7, 1)]
    views[1][1]["frame_index"], views[1][1]["view_index"] = torch.tensor([7]), 1     # host values
    vis.visualize(*views[0])                                                           # allocates the ring
    vis.flush()
    torch.cuda.synchronize()
    try:
        torch.cuda.set_sync_debug_mode("error")
        for _ in range(3):
            for out, batch in views:
                vis.visualize(out, batch)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    vis.flush()
    want = O.frame(rgb, mask, 540, 540)
    for v in (0, 1):
        got = cv2.imread(str(tmp_path / "data" / "perform" / "vis" / "0" / ("frame0007_view%04d.png" % v)), cv2.IMREAD_UNCHANGED)
        assert np.array_equal(got, want)


def test_many_views_through_the_ring(monkeypatch, tmp_path):
    """More views than slots, two sizes, device and host tensors: every file has its own view's bytes."""
    pytest.importorskip("cv2")
    monkeypatch.chdir(tmp_path)
    vis = _visualizer("demo")
    want = {}
    for i in range(11):
        H, W = (64, 48) if i < 7 else (100, 120)
        _cfg(H, W, i % 2)
        rgb, mask = VC.random_view(H, W, 100 + i)
        vis.visualize(*_view(rgb, mask, i // 4, i, DEV if i % 3 else torch.device("cpu")))
        want[(i // 4, i)] = O.frame(rgb, mask, H, W, i % 2)
    vis.flush()
    for (f, v), frame in want.items():
        p = tmp_path / "data" / "render" / "vis" / ("frame_%04d" % f) / ("%04d.png" % v)
        assert open(p, "rb").read() == _png_bytes(frame, tmp_path / "want.png"), (f, v)


def _scene_from_item(item, seed=313):
    from oracle import synth
    coord, out_sh = np.asarray(item["coord"]), np.asarray(item["out_sh"])
    volumes, _ = synth.make_volumes(coord, out_sh, seed)
    weights = synth.trained_like_rescale(synth.make_weights(seed, 60), volumes, seed)
    return {"volumes": volumes, "weights": weights, "voxel_size": [0.005, 0.005, 0.005]}


def _rotate_item(g, v):
    """The rotate drop-in's item for golden view v, over a base that returns the golden's upstream values."""
    from neuralbody_b200.lib.datasets.light_stage import rotate_smpl_dataset as drop
    x = g["views"][v]

    class Base:
        K = x["K"]
        render_w2c = [x["RT"]]

        def prepare_input(self, i, index):
            assert (i, index) == (int(x["frame_index"]), v)
            return x["coord"], x["out_sh"], x["can_bounds"], x["bounds"], x["R"], x["Th"]

    ds = drop.make_dataset_class(Base, cv2=types.SimpleNamespace(Rodrigues=lambda R: (R,)))()
    return ds[v]


def _collate(item, dev):
    """default_collate of one item, then upstream's visualize loop: every key but 'meta' to the device."""
    batch = {}
    for k, val in item.items():
        if k == "meta":
            batch[k] = {m: torch.as_tensor(np.asarray(a))[None] for m, a in val.items()}
        else:
            batch[k] = torch.as_tensor(np.asarray(val))[None].to(dev)
    return batch


def _renderer(mod, scene, precision="tc_fp16x3"):
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.networks.make_network import load_source
    from gpu_utils import make_net_and_renderer
    from conftest import ROOT
    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.raw_noise_std = 64, 0.0, False, 0
    cfg.render_precision, cfg.render_volume_dtype, cfg.chunk, cfg.render_skip_empty = precision, "auto", 0, True
    net, _ = make_net_and_renderer(scene)
    net.train(False)
    path = os.path.join(ROOT, "neuralbody_b200", "lib", "networks", "renderer", mod + ".py")
    return load_source("neuralbody_b200.lib.networks.renderer." + mod, path).Renderer(net)


@pytest.mark.parametrize("precision", ["fp32", "tc_fp16x3"])
def test_rotate_item_renders_upstreams_rays(precision):
    """A rotate drop-in item (the camera) renders the maps of upstream's item (its host rays), bit for bit, with the same
    mask_at_box."""
    g = VC.load_rotate_golden()
    from neuralbody_b200.lib.config import cfg
    for v in VC.ROTATE_VIEWS:
        x = g["views"][v]
        item = _rotate_item(g, v)
        assert "ray_o" not in item and item["cam_RT"] is x["RT"] and item["can_bounds"] is x["can_bounds"]
        ren = _renderer("if_nerf_renderer", _scene_from_item(item), precision)
        cfg.H, cfg.W, cfg.ratio = 2 * g["H"], 2 * g["W"], 0.5
        cam = _collate(item, DEV)
        rays = _collate({k: item[k] for k in VC.ROTATE_KEYS}, DEV)
        for k in ("ray_o", "ray_d", "near", "far"):
            rays[k] = torch.from_numpy(x[k])[None].to(DEV)
        with torch.no_grad():
            got, want = ren.render(cam), ren.render(rays)
        assert np.array_equal(cam["mask_at_box"][0].cpu().numpy(), x["mask_at_box"])
        for k in want:
            a, b = got[k].cpu().numpy(), want[k].cpu().numpy()
            assert a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32)), (v, k)
        assert float(want["acc_map"].max()) > 0, v                    # the rays reach the body


def test_render_then_visualize_writes_upstreams_files(monkeypatch, tmp_path):
    """End to end on synthetic scenes: the rotate drop-in item through the plain renderer and if_nerf_demo's drop-in, and
    a novel-view camera batch through the _mmsk renderer and if_nerf_perform's drop-in; each PNG is at upstream's path
    and has the bytes of cv2.imwrite of the restatement's frame of the same maps."""
    pytest.importorskip("cv2")
    from neuralbody_b200.lib.config import cfg
    from tools import mesh_mono_case as MM
    from tools import demo_case as DC
    monkeypatch.chdir(tmp_path)
    g = VC.load_rotate_golden()
    # rotate-SMPL: plain renderer, if_nerf_demo
    item = _rotate_item(g, 17)
    ren = _renderer("if_nerf_renderer", _scene_from_item(item))
    cfg.H, cfg.W, cfg.ratio, cfg.white_bkgd, cfg.exp_name = 2 * g["H"], 2 * g["W"], 0.5, False, "rot"
    vis = _visualizer("demo")
    batch = _collate(item, DEV)
    with torch.no_grad():
        out = ren.render(batch)
        vis.visualize(out, batch)
    vis.flush()
    want = O.frame(out["rgb_map"][0].cpu().numpy(), batch["mask_at_box"][0].cpu().numpy(), g["H"], g["W"])
    got = open(tmp_path / VC.reference_path("demo", "rot", 0, 17), "rb").read()
    assert got == _png_bytes(want, tmp_path / "want.png")
    # novel view: _mmsk renderer with mask views, if_nerf_perform
    scene = MM.make_scene(0.3)
    H, W = 100, 75
    K = MM.get_camera(MM.camera_pkl(scene, H, W))["K"]
    msk = (MM.silhouette(scene, K, H, W, 2) != 0).astype(np.uint8)
    ren = _renderer("if_nerf_renderer_mmsk", scene)
    cfg.H, cfg.W, cfg.ratio, cfg.white_bkgd, cfg.exp_name = H, W, 1.0, True, "nv"
    RT = np.eye(4)
    RT[:3, 3] = (0.004, -0.002, 0.01)
    cb = scene["can_bounds"][0].numpy()
    batch = {k: scene[k].to(DEV) for k in ("coord", "out_sh", "bounds", "R", "Th", "latent_index")}
    batch.update({"msks": torch.from_numpy(msk)[None, None].to(DEV),
                  "RT": torch.from_numpy(RT[:3].astype(np.float32))[None, None].to(DEV),
                  "Ks": torch.from_numpy(K.astype(np.float32))[None, None].to(DEV),
                  "cam_RT": torch.from_numpy(RT)[None].to(DEV), "cam_K": torch.from_numpy(K)[None].to(DEV),
                  "can_bounds": torch.from_numpy(cb)[None].to(DEV),
                  "frame_index": torch.tensor([5]).to(DEV), "view_index": torch.tensor([2]).to(DEV)})
    vis = _visualizer("perform")
    with torch.no_grad():
        out = ren.render(batch)
        vis.visualize(out, batch)
    vis.flush()
    mask = batch["mask_at_box"][0].cpu().numpy()
    assert np.array_equal(mask, DC.image_rays_numpy(RT, K, cb, H, W)[4])
    want = O.frame(out["rgb_map"][0].cpu().numpy(), mask, H, W, True)
    got = open(tmp_path / VC.reference_path("perform", "nv", 5, 2), "rb").read()
    assert got == _png_bytes(want, tmp_path / "want.png")
