"""Helpers for the GPU parity tests: drive the product path (Renderer.render -> ctypes -> C ABI)."""
import numpy as np
import torch

from neuralbody_b200.lib.config import cfg
from neuralbody_b200.lib.networks.make_network import make_network
from neuralbody_b200.lib.networks.renderer.make_renderer import make_renderer

BATCH_KEYS = ("coord", "out_sh", "bounds", "R", "Th", "latent_index", "ray_o", "ray_d", "near", "far")


def make_net_and_renderer(scene, device="cuda:0"):
    cfg.num_train_frame = int(scene["weights"]["latent.weight"].shape[0])
    cfg.voxel_size = list(scene["voxel_size"])
    net = make_network(cfg)
    missing, unexpected = net.load_state_dict(scene["weights"], strict=False)
    assert not unexpected and all(k.startswith("c.") for k in missing), (missing, unexpected)
    net = net.to(device)
    net.set_feature_volume([v.to(device) for v in scene["volumes"]])
    return net, make_renderer(cfg, net)


def render_product(scene, n_samples=64, perturb=0.0, training=False, white_bkgd=False, t_rand=None,
                   precision="fp32", device="cuda:0", want_raw=False, chunk=0, renderer=None, net=None, skip_empty=True,
                   masks=None):
    """Render `scene` through the public API on the GPU; returns dict of CPU tensors."""
    cfg.N_samples = int(n_samples)
    cfg.perturb = float(perturb)
    cfg.white_bkgd = bool(white_bkgd)
    cfg.raw_noise_std = 0
    cfg.render_precision = precision
    cfg.render_volume_dtype = "auto"
    cfg.chunk = int(chunk)
    cfg.render_skip_empty = bool(skip_empty)
    if renderer is None:
        net, renderer = make_net_and_renderer(scene, device)
    net.train(training)
    batch = {k: scene[k].to(device) for k in BATCH_KEYS}
    if masks is not None:   # f-1: the masked renderer plugin, selected by path like any other renderer
        import os
        from neuralbody_b200.lib.networks.make_network import load_source
        here = os.path.dirname(os.path.abspath(__file__))
        single = "R0_snap" in masks          # if_clight_renderer_msk (one snapshot view) vs _mmsk (nv training views)
        mod = "if_nerf_renderer_msk" if single else "if_nerf_renderer_mmsk"
        path = os.path.join(here, "..", "neuralbody_b200", "lib", "networks", "renderer", mod + ".py")
        mren = load_source("neuralbody_b200.lib.networks.renderer." + mod, os.path.abspath(path)).Renderer(net)
        cfg.H, cfg.W, cfg.ratio = int(masks["mask_H"]), int(masks["mask_W"]), 1.0
        batch.update({k: masks[k].to(device) for k in (("R0_snap", "Th0_snap", "RT", "K", "msk") if single else ("RT", "Ks", "msks"))})
        with torch.no_grad():
            out = mren.render(batch)
        torch.cuda.synchronize()
        return {k: v.detach().cpu() for k, v in out.items()}
    if t_rand is not None or want_raw:
        sp_input = renderer.prepare_sp_input(batch)
        vol = net.encode_sparse_voxels(sp_input)
        with torch.no_grad():
            out = renderer.render_rays(batch["ray_o"], batch["ray_d"], batch["near"], batch["far"], vol, sp_input,
                                       t_rand=None if t_rand is None else t_rand.to(device), want_raw=want_raw)
    else:
        with torch.no_grad():
            out = renderer.render(batch)
    torch.cuda.synchronize()
    return {k: v.detach().cpu() for k, v in out.items()}


def backward_kernel_names(loss, settle_s=0.1):
    """Names of the CUDA kernels and memsets `loss.backward()` enqueues, from torch.profiler.  The profiler keeps only the
    device activities that start inside its capture window, whose start is a host timestamp taken when the trace starts;
    the device timestamps are converted to that clock.  A kernel launched right after the start can be stamped just before
    it and is dropped: on a busy host the first kernels of a backward (its loss-gradient multiplies, the gradient zeroing)
    were seen missing.  So the backward is launched `settle_s` after the trace started, on an idle device."""
    import time
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time.sleep(settle_s)
        loss.backward()
        torch.cuda.synchronize()
    return {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}


def compare(out, gold, atol_main, atol_weights=None, nan_mismatch_frac=0.0, label=""):
    """max-abs comparison of the five outputs.  rgb_map / depth_map / acc_map / weights: absolute;
    disp_map = 1/(depth/acc) is ill-conditioned where acc ~ 0, so it is compared relatively on rays
    with acc > 1e-2, and its NaN pattern (acc == 0 rays) must agree."""
    report = {}
    for k in ("rgb_map", "depth_map", "acc_map"):
        d = float(np.abs(out[k].numpy() - np.asarray(gold[k])).max())
        report[k] = d
        assert d <= atol_main, "%s %s max abs diff %.3e > %.1e" % (label, k, d, atol_main)
    if "weights" in out:
        d = float(np.abs(out["weights"].numpy() - np.asarray(gold["weights"])).max())
        report["weights"] = d
        assert d <= (atol_weights or atol_main), "%s weights max abs diff %.3e" % (label, d)
    a, b = out["disp_map"].numpy(), np.asarray(gold["disp_map"])
    nan_a, nan_b = np.isnan(a), np.isnan(b)
    mism = float((nan_a != nan_b).mean())
    report["disp_nan_mismatch"] = mism
    assert mism <= nan_mismatch_frac, "%s disp NaN pattern differs on %.4f of rays" % (label, mism)
    ok = (~nan_a) & (~nan_b) & (np.asarray(gold["acc_map"]) > 1e-2)
    if ok.any():
        rel = float((np.abs(a[ok] - b[ok]) / np.abs(b[ok])).max())
        report["disp_rel"] = rel
        assert rel <= max(50 * atol_main, 1e-3), "%s disp rel diff %.3e" % (label, rel)
    return report
