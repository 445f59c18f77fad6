"""GPU: the training wrapper drop-in (lib/train/trainers/if_nerf_clight.py) and its device losses (nb_image_loss_fwd /
_bwd) against upstream's expression torch.mean((rgb_map[mask] - rgb[mask]) ** 2) (+ the unmasked rgb0 term):
  - the loss within 1e-6 relative of float64, the same bits on every call; an empty mask gives NaN and zero gradients;
  - the rgb_map / rgb0 cotangents bit for bit with CUDA autograd through upstream's expression, for any loss cotangent;
  - a full training step through the wrapper hands the renderer's backward the same cotangents as upstream's wrapper, bit
    for bit, so every parameter and volume gradient is upstream's up to the order of the renderer's float atomicAdds, which
    varies from run to run for upstream's expression as well;
  - the wrapper's forward and loss.backward() run under torch.cuda.set_sync_debug_mode('error'), where upstream's
    boolean index raises;
  - under no_grad, on a test-split item of this package's datasets, the stats are upstream's."""
import os

import numpy as np
import pytest
import torch

import gpu_utils as G
from conftest import ROOT
from test_image_loss_cpu import _case, restate_cotangent

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _upstream_mse(x, y, mask=None):
    return torch.mean((x[mask] - y[mask]) ** 2) if mask is not None else torch.mean((x - y) ** 2)


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("kind", ["all", "partial", "empty"])
@pytest.mark.parametrize("n", [1024, 70001])
@pytest.mark.parametrize("mask_dtype", [torch.bool, torch.uint8])
def test_loss_is_float64s_and_reproducible(B, kind, n, mask_dtype):
    from neuralbody_b200.image_loss import image_mse
    pred, gt, mask = _case(B, n, kind, 3 * B + n)
    x, y = torch.from_numpy(pred).to(DEV), torch.from_numpy(gt).to(DEV)
    m = torch.from_numpy(mask).to(DEV).to(mask_dtype)
    loss, count = image_mse(x, y, m, with_count=True)
    again = [image_mse(x, y, m) for _ in range(3)]
    d = (pred.astype(np.float64) - gt)[mask]
    assert int(count) == d.size
    if kind == "empty":
        assert torch.isnan(loss) and all(torch.isnan(a) for a in again)
    else:
        ref = float(np.mean(d ** 2))
        assert abs(float(loss) - ref) <= 1e-6 * ref
        assert all(torch.equal(a.view(torch.int32), loss.view(torch.int32)) for a in again)
    l0 = image_mse(x, y)
    ref0 = float(np.mean((pred.astype(np.float64) - gt) ** 2))
    assert abs(float(l0) - ref0) <= 1e-6 * ref0


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("kind", ["all", "partial", "empty"])
@pytest.mark.parametrize("g", [1.0, 0.37, -2.5e-3])
def test_cotangents_are_cuda_autograds(B, kind, g):
    from neuralbody_b200.image_loss import image_mse
    pred, gt, mask = _case(B, 1024, kind, 5 * B)
    y, m = torch.from_numpy(gt).to(DEV), torch.from_numpy(mask).to(DEV)
    gl = torch.tensor(g, device=DEV)
    for masked in (True, False):
        mm = m if masked else None
        a = torch.from_numpy(pred).to(DEV).requires_grad_(True)
        b = torch.from_numpy(pred).to(DEV).requires_grad_(True)
        image_mse(a, y, mm).backward(gl)
        _upstream_mse(b, y, mm).backward(gl)
        assert torch.equal(a.grad.view(torch.int32), b.grad.view(torch.int32)), (kind, g, masked)
        if masked and kind == "empty":
            assert not a.grad.view(torch.int32).any()          # +0.0 everywhere, as upstream's scatter into zeros
    # the CPU restatement of the rounding is the kernel's too
    n_set = 3 * int(mask.sum())
    want = restate_cotangent(pred, gt, mask, np.float32(1.0), n_set)
    a = torch.from_numpy(pred).to(DEV).requires_grad_(True)
    image_mse(a, y, m).backward()
    assert torch.equal(a.grad.cpu().view(torch.int32), want.view(torch.int32))


# ----------------------------------------------------------------------------------------------- the wrapper, end to end
def _wrapper_module():
    from neuralbody_b200.lib.networks.make_network import load_source
    path = os.path.join(ROOT, "neuralbody_b200", "lib", "train", "trainers", "if_nerf_clight.py")
    return load_source("lib.train.trainers.if_nerf_clight", path)


def _setup(B, importance, precision, seed=0):
    from oracle import synth
    from neuralbody_b200.lib.config import cfg
    scene = synth.make_scene(H=32, W=32, scale=0.25, all_hit=True)
    net, _ = G.make_net_and_renderer(scene, DEV)
    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.raw_noise_std, cfg.chunk = 64, 0.0, False, 0, 0
    cfg.render_precision, cfg.render_volume_dtype, cfg.render_skip_empty = "tc_fp16x3", "auto", True
    cfg.render_importance, cfg.render_train_precision, cfg.render_return_weights = importance, precision, True
    net.train()
    nt = int(scene["weights"]["latent.weight"].shape[0])
    batch = {k: torch.cat([scene[k]] * B, 0).to(DEV) for k in G.BATCH_KEYS if k != "latent_index"}
    batch["latent_index"] = (torch.arange(B) % nt).to(DEV)
    n = batch["ray_o"].shape[1]
    g = torch.Generator().manual_seed(seed)
    batch["rgb"] = torch.rand((B, n, 3), generator=g).to(DEV)
    batch["mask_at_box"] = (torch.rand((B, n), generator=g) < 0.8).to(DEV)
    vols = [torch.cat([v] * B, 0).to(DEV).requires_grad_(True) for v in scene["volumes"]]
    net.set_feature_volume(vols)
    wrapper = _wrapper_module().NetworkWrapper(net)
    return scene, net, wrapper, batch, vols


def _record_cotangents(ren):
    seen = []
    orig = ren._launch_bwd

    def rec(call, d_rgb, *a, **k):
        seen.append(None if d_rgb is None else d_rgb.detach().clone())
        return orig(call, d_rgb, *a, **k)
    ren._launch_bwd = rec
    return seen


def _grads(net, vols):
    out = {n: (None if p.grad is None else p.grad.clone()) for n, p in net.named_parameters()}
    out.update({"volume%d" % i: v.grad.clone() for i, v in enumerate(vols)})
    for p in net.parameters():
        p.grad = None
    for v in vols:
        v.grad = None
    return out


@pytest.mark.parametrize("importance", [0, 64])
@pytest.mark.parametrize("precision", ["tc_tf32x3", "fp32"])
def test_training_step_gradients_are_upstreams(importance, precision):
    """B = 2 frames, a partial mask: one step through the wrapper, then two through upstream's expression on the same
    renderer and batch."""
    scene, net, wrapper, batch, vols = _setup(2, importance, precision)
    ren = wrapper.renderer
    seen = _record_cotangents(ren)
    ret, loss, stats, image_stats = wrapper(batch)
    assert set(stats) == ({"img_loss", "loss"} | ({"img_loss0"} if importance else set())) and image_stats == {}
    loss.backward()
    mine, mine_d = _grads(net, vols), list(seen)
    ups = []
    for _ in range(2):
        del seen[:]
        r = ren.render(batch)
        m = batch["mask_at_box"]
        u_loss = 0
        u_img = torch.mean((r["rgb_map"][m] - batch["rgb"][m]) ** 2)
        u_loss += u_img
        if "rgb0" in r:
            u_img0 = torch.mean((r["rgb0"] - batch["rgb"]) ** 2)
            assert abs(stats["img_loss0"].item() - u_img0.item()) <= 2e-6 * u_img0.item()
            u_loss += u_img0
        u_loss.backward()
        ups.append((_grads(net, vols), list(seen)))
        assert abs(stats["img_loss"].item() - u_img.item()) <= 2e-6 * u_img.item()
    (u1, u1_d), (u2, u2_d) = ups
    assert len(mine_d) == len(u1_d) == len(u2_d) == (2 if importance else 1)
    for a, b in zip(mine_d, u1_d):      # what the drop-in controls: the cotangents the renderer's backward receives
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    for k in mine:
        # from equal cotangents the renderer's backward gives equal gradients up to the order of its float atomicAdds, which
        # changes from run to run (upstream against upstream differs in the last bits too): both pairs get the same bound
        a, b, b2 = mine[k], u1[k], u2[k]
        assert (a is None) == (b is None) == (b2 is None), k
        if a is None:
            continue
        tol = 1e-4 * float(b.abs().max()) + 1e-12
        assert float((a - b).abs().max()) <= tol and float((b2 - b).abs().max()) <= tol, k


@pytest.mark.parametrize("importance", [0, 64])
def test_step_does_not_synchronise(importance):
    """After prepare_sp_input (whose .tolist() is upstream's one wait per frame), the wrapper's forward and loss.backward()
    enqueue without a host synchronisation; upstream's expression on the same render raises in this mode."""
    scene, net, wrapper, batch, vols = _setup(1, importance, "tc_tf32x3")
    ren = wrapper.renderer
    _, loss, _, _ = wrapper(batch)              # warm-up: caches, packs and pools
    loss.backward()
    sp = ren.prepare_sp_input(batch)
    ren.prepare_sp_input = lambda b: sp
    torch.cuda.synchronize()
    try:
        torch.cuda.set_sync_debug_mode("error")
        _, loss, stats, _ = wrapper(batch)
        loss.backward()
        r = ren.render(batch)
        with pytest.raises(RuntimeError):
            torch.mean((r["rgb_map"][batch["mask_at_box"]] - batch["rgb"][batch["mask_at_box"]]) ** 2)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert torch.isfinite(loss) and net.fc_0.weight.grad is not None


def test_empty_mask_gives_nan_loss_and_zero_grads():
    scene, net, wrapper, batch, vols = _setup(1, 0, "tc_tf32x3")
    batch["mask_at_box"] = torch.zeros_like(batch["mask_at_box"])
    _, loss, stats, _ = wrapper(batch)
    loss.backward()
    assert torch.isnan(stats["img_loss"]) and torch.isnan(loss)
    for name, p in net.named_parameters():
        assert p.grad is None or not p.grad.any(), name
    assert all(not v.grad.any() for v in vols)


def _device_item(scene, H, W, split):
    """A batch as this package's multi_view_dataset drop-in ships it (dataset_image_steps: 'device'): the image and the
    camera instead of the rays; a narrow view, so that every pixel's ray hits the box."""
    from oracle import synth
    from neuralbody_b200 import rays
    cb = scene["can_bounds"][0].numpy().astype(np.float32)
    Ks, RTs = synth.training_cameras(0.5 * (cb[0] + cb[1]).astype(np.float64), n_cams=1, distance=3.0, f=40.0 * H, H=H, W=W)
    k_kind, cam = rays.train_camera(Ks[0], RTs[0][:3, :3].copy(), RTs[0][:3, 3:4].copy(), cb)
    g = torch.Generator().manual_seed(3)
    batch = {k: scene[k].to(DEV) for k in ("coord", "out_sh", "bounds", "R", "Th", "latent_index")}
    batch["img"] = torch.rand((1, H, W, 3), generator=g).to(DEV)
    meta = {"train_cam": torch.from_numpy(cam)[None], "train_k_kind": torch.tensor([k_kind])}
    if split == "train":
        from neuralbody_b200 import capi
        batch["ray_class"] = torch.full((1, H, W), capi.NB_TRAIN_CLASS_BODY | capi.NB_TRAIN_CLASS_BOUND, dtype=torch.uint8,
                                        device=DEV)
        meta.update({"N_rand": torch.tensor([256]), "body_sample_ratio": torch.tensor([0.5]),
                     "face_sample_ratio": torch.tensor([0.0])})
    batch["meta"] = meta
    return batch


@pytest.mark.parametrize("split", ["train", "test"])
def test_device_items_train_and_validate(split):
    """This package's items: split 'train' trains (the renderer samples the rays and writes rgb / mask_at_box before the
    loss reads them); split 'test' under no_grad, as Trainer.val runs it, returns upstream's stats of the view."""
    scene, net, wrapper, _, vols = _setup(1, 0, "tc_tf32x3")
    batch = _device_item(scene, 16, 16, split)
    if split == "train":
        _, loss, stats, _ = wrapper(batch)
        loss.backward()
        m = batch["mask_at_box"]
        assert m.shape == (1, 256) and bool(m.all()) and batch["rgb"].shape == (1, 256, 3)
        assert torch.isfinite(loss) and net.fc_0.weight.grad is not None
        return
    net.eval()
    with torch.no_grad():
        ret, loss, stats, _ = wrapper(batch)
    m = batch["mask_at_box"]
    assert m.shape == (1, 256) and bool(m.all()), "the view must lie inside the box for upstream's index to work"
    want = torch.mean((ret["rgb_map"][m] - batch["rgb"][m]) ** 2)
    assert set(stats) == {"img_loss", "loss"}
    assert abs(float(stats["img_loss"]) - float(want)) <= 2e-6 * float(want)
    assert torch.equal(stats["loss"], stats["img_loss"] + 0)
