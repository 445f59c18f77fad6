"""nb_item_images: the training datasets' image steps after decoding on the GPU, bit for bit with the numpy restatement
(oracle/item_images.py, pinned to OpenCV by test_item_images_cpu) and with OpenCV's outputs in the goldens; a batch of
'device' items renders and trains as the 'host' items do."""
import numpy as np
import pytest
import torch

from oracle import item_images as O
from tools import item_images_case as IC

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _run(items, H, W, bkgd=0, rule=0, bounds=None):
    from neuralbody_b200 import images
    cams = [images.item_camera(K, D) for _, _, K, D in items]
    img_u8 = torch.from_numpy(np.stack([it[0] for it in items])).to(DEV)
    msk_u8 = torch.from_numpy(np.stack([it[1] for it in items])).to(DEV)
    bound = torch.from_numpy(np.stack(bounds)).to(DEV) if bounds is not None else None
    img, msk, cmap = images.item_images(img_u8, msk_u8, np.stack([c for _, c in cams]), cams[0][0], H, W, bkgd, rule, bound)
    torch.cuda.synchronize()
    return img.cpu().numpy(), msk.cpu().numpy(), None if cmap is None else cmap.cpu().numpy()


def _bound(H, W, seed):
    rng = np.random.RandomState(seed)
    b = np.zeros((H, W), np.uint8)
    y0, x0 = rng.randint(0, H // 4), rng.randint(0, W // 4)
    b[y0:y0 + H // 2, x0:x0 + W // 2] = 1
    return b


def _check(got, want, tie, label):
    img, msk, cmap = got
    wimg, wmsk, wcmap = want
    bad = (img.view(np.uint32) != wimg.view(np.uint32)).any(-1) | (msk != wmsk)
    if wcmap is not None:
        bad |= cmap != wcmap
    print("%s: %d flagged pixels, %d of them differ" % (label, tie.sum(), (bad & tie).sum()))
    assert not (bad & ~tie).any(), "%s: %d pixels differ outside flagged ties" % (label, (bad & ~tie).sum())


FULL = [(1024, 1024, 0.5, "k1", 1, 1), (1080, 1080, 0.5, "rational8", 2, 2), (1080, 1080, 1.0, "tangential", 1, 2),
        (1000, 1002, 1.0, "zero", 0, 1)]


@pytest.mark.parametrize("case", FULL, ids=["%dx%d_r%g_%s" % c[:4] for c in FULL])
def test_full_size_equals_the_restatement(case):
    H0, W0, ratio, dist, bkgd, rule = case
    it = IC.case(H0, W0, dist, seed=H0 + W0)
    H, W = int(H0 * ratio), int(W0 * ratio)
    bound = _bound(H, W, 0)
    img, msk, cmap, tie = O.item_images(*it, H, W, bkgd, rule, bound)
    _check(_run([it], H, W, bkgd, rule, [bound]), (img[None], msk[None], cmap[None]), tie[None], str(case))


def test_goldens_equal_opencv():
    for c, g in enumerate(IC.load_golden()):
        H0, W0 = g["msk_u8"].shape
        H, W = int(H0 * g["ratio"]), int(W0 * g["ratio"])
        it = (g["img_u8"], g["msk_u8"], g["K"], g["D"])
        tie = O.item_images(*it, H, W, int(g["bkgd"]))[3]
        _check(_run([it], H, W, int(g["bkgd"])), (g["img"][None], g["msk"][None], None), tie[None], "golden %d" % c)


def test_batch_of_two_cameras():
    """Two items with different cameras and distortion models in one launch: each is its own restatement."""
    a = IC.case(540, 720, "k1", 3)
    b = list(IC.case(540, 720, "tangential", 4))
    b[2] = b[2].copy()
    b[2][0, 0] *= 0.93
    b[2][1, 2] += 11.3
    b[3] = np.concatenate([b[3], np.zeros((1, 1))])           # the same model as five coefficients
    bounds = [_bound(270, 360, 1), _bound(270, 360, 2)]
    got = _run([a, tuple(b)], 270, 360, 2, 2, bounds)
    for n, (it, bd) in enumerate(zip((a, b), bounds)):
        img, msk, cmap, tie = O.item_images(*it, 270, 360, 2, 2, bd)
        _check(tuple(x[n:n + 1] for x in got), (img[None], msk[None], cmap[None]), tie[None], "item %d" % n)
    assert not np.array_equal(got[0][0], got[0][1])


# ----------------------------------------------------------------------------- the renderer on 'device' items
def _scene_item(split, bkgd_white=False):
    """A People-Snapshot-like item pair from the mesh scene: the decoded image and mask at 2x with a mild distortion,
    the host item's processed image, mask and class map (OpenCV's steps, as the restatement) and the device item's keys."""
    from tools import mesh_mono_case as MM
    from neuralbody_b200.lib.datasets import train_item
    scene = MM.make_scene(0.3)
    H, W = 100, 76
    K2 = MM.get_camera(MM.camera_pkl(scene, H, W))["K"].astype(np.float64)
    K2[:2] *= 2
    msk0 = (MM.silhouette(scene, K2, 2 * H, 2 * W, 2) != 0).astype(np.uint8) * 255
    rng = np.random.RandomState(0)
    img_u8 = rng.randint(0, 256, (2 * H, 2 * W, 3)).astype(np.uint8)
    D = np.array([0.02, -0.01, 0.0005, 0.0003, 0.])
    img, msk, _, _ = O.item_images(img_u8, msk0, K2, D, H, W, 2 if bkgd_white else 1)
    Ks = K2.astype(np.float32)
    Ks[:2] = Ks[:2] * np.float32(0.5)
    ys, xs = np.nonzero(msk)
    bound = np.zeros((H, W), np.uint8)
    bound[max(ys.min() - 6, 0):ys.max() + 7, max(xs.min() - 6, 0):xs.max() + 7] = 1
    R, T = np.eye(3), np.zeros((3, 1))
    cb = scene["can_bounds"][0].numpy().astype(np.float32)
    host = train_item.camera_fields(Ks, R, T, cb, 1024, 0.5, 0.0) if split == "train" else \
        train_item.camera_fields(Ks, R, T, cb)
    dev_keys, meta = train_item.device_fields(img_u8, msk0, K2, D, H, W, True, bkgd_white, True,
                                              train_item.CLASS_SNAPSHOT if split == "train" else None,
                                              bound if split == "train" else None)
    host_keys = {"img": img, "msk": msk}
    if split == "train":
        host_keys["ray_class"] = train_item.class_map_snapshot(msk, bound)
    return scene, host, host_keys, dev_keys, meta


def _batch(scene, host, keys, meta=None):
    from gpu_utils import BATCH_KEYS
    b = {k: scene[k].to(DEV) for k in BATCH_KEYS if k not in ("ray_o", "ray_d", "near", "far")}
    b.update({k: torch.from_numpy(np.asarray(v))[None].to(DEV) for k, v in keys.items()})
    m = {k: torch.as_tensor(np.asarray(v))[None] for k, v in host["meta"].items()}
    if meta is not None:
        m.update({k: torch.as_tensor(np.asarray(v))[None] for k, v in meta.items()})
    b["meta"] = m
    return b


def test_training_step_from_device_items_equals_the_host_items():
    """render -> loss -> backward from a 'device' batch (nb_item_images, then the sampler) equals the step from the
    'host' batch with the same Philox key: the processed image, mask and class map bit for bit, then the outputs and the
    loss, and the gradients to the run-to-run spread of the backward's atomic accumulation."""
    from neuralbody_b200.lib.config import cfg
    from gpu_utils import make_net_and_renderer
    scene, host, host_keys, dev_keys, meta = _scene_item("train")
    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.raw_noise_std, cfg.chunk = 64, 1.0, False, 0, 0
    cfg.render_train_precision = "tc_tf32x3"
    outs = []
    for keys, extra in ((host_keys, None), (dev_keys, meta)):
        net, ren = make_net_and_renderer(scene)
        net.train(True)
        batch = _batch(scene, host, keys, extra)
        torch.manual_seed(7)
        ret = ren.render(batch)
        mask = batch["mask_at_box"]
        loss = torch.mean((ret["rgb_map"][mask] - batch["rgb"][mask]) ** 2)
        loss.backward()
        torch.cuda.synchronize()
        outs.append((batch, {k: v.detach().cpu() for k, v in ret.items()}, loss.item(),
                     [p.grad.detach().cpu().clone() for p in net.parameters() if p.grad is not None]))
    (b0, o0, l0, g0), (b1, o1, l1, g1) = outs
    for k in ("img", "msk", "ray_class", "rgb", "ray_o", "ray_d", "near", "far"):
        assert torch.equal(b0[k].cpu(), b1[k].cpu()), k
    same = lambda a, b: a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert l0 == l1
    for k in o0:
        assert same(o0[k], o1[k]), k
    assert len(g0) == len(g1) > 0
    for a, b in zip(g0, g1):
        scale = float(a.abs().max()) or 1.0
        assert float((a - b).abs().max()) <= 1e-4 * scale


def test_test_split_rays_match_the_host_item():
    from gpu_utils import make_net_and_renderer
    scene, host, host_keys, dev_keys, meta = _scene_item("test", bkgd_white=True)
    _, ren = make_net_and_renderer(scene)
    got = []
    for keys, extra in (({"img": host_keys["img"]}, None), (dev_keys, meta)):
        batch = _batch(scene, host, keys, extra)
        rays = ren.camera_rays(batch)
        torch.cuda.synchronize()
        got.append([r.cpu() for r in rays] + [batch["rgb"].cpu(), batch["mask_at_box"].cpu()])
    for a, b in zip(*got):
        assert torch.equal(a, b)


def test_empty_body_list_raises_value_error():
    """A 'device' item whose mask is empty inside the bound: upstream's item raises ValueError; here the sampler's status
    does, after the render's existing synchronisation."""
    from gpu_utils import make_net_and_renderer
    scene, host, _, dev_keys, meta = _scene_item("train")
    dev_keys = dict(dev_keys, msk_u8=np.zeros_like(dev_keys["msk_u8"]))
    _, ren = make_net_and_renderer(scene)
    batch = _batch(scene, host, dev_keys, meta)
    with pytest.raises(ValueError):
        ren.render(batch)
