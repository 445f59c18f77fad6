"""What the fine pass costs on a masked demo view: the novel-view loop's render (the `_mmsk` renderer, four mask views) of one
512 x 512 orbit view, coarse only (`render_importance: 0`) against coarse + fine (`render_importance: 128`), alternated
view by view in one process; medians.

    python -m tools.bench_demo_importance [--views 20] [--precision tc_fp16x3]

The view is the first multi-view orbit camera of tests/golden/demo_orbit_s512.npz over synth's full-size body; the four
mask views are the body's silhouettes from cameras around it (oracle.synth.make_mask_views at the view's size, so they
cut the body where the views disagree).  The scene supplies its feature volumes, so the sparse-convolution encode is
excluded, and the rays are built once, on the device.  Reported per mode: the host time of get_pixel_value until the
device is done (ms per view), the device time between CUDA events around it, and from one extra counting run per mode
the samples the classifier listed for the decoder in each pass (the rest were masked out or in empty space)."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools import demo_case as DC  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=20)
    ap.add_argument("--precision", default="tc_fp16x3")
    ap.add_argument("--importance", type=int, default=128)
    args = ap.parse_args()
    from neuralbody_b200 import rays
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.networks.make_network import load_source
    from oracle import synth
    from tools import mesh_mono_case as MM
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from gpu_utils import make_net_and_renderer
    z = np.load(DC.ORBIT)
    H, W = (int(v) for v in z["mv_HW"])
    scene = MM.make_scene(1.0)
    cb = scene["can_bounds"][0].numpy()
    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.raw_noise_std = 64, 0.0, False, 0
    cfg.render_precision, cfg.render_volume_dtype, cfg.chunk, cfg.render_skip_empty = args.precision, "auto", 0, True
    cfg.H, cfg.W, cfg.ratio = H, W, 1.0
    net, _ = make_net_and_renderer(scene)
    net.train(False)
    mod = load_source("neuralbody_b200.lib.networks.renderer.if_nerf_renderer_mmsk",
                      os.path.join(ROOT, "neuralbody_b200", "lib", "networks", "renderer", "if_nerf_renderer_mmsk.py"))
    ren = mod.Renderer(net)
    dev = torch.device("cuda:0")
    masks = synth.make_mask_views(scene, nv=4, H=H, W=W, radius=3)
    batch = {k: scene[k].to(dev) for k in ("coord", "out_sh", "bounds", "R", "Th", "latent_index")}
    batch.update({k: masks[k].to(dev) for k in ("RT", "Ks", "msks")})
    ro, rd, near, far, _ = rays.camera_image_rays(z["mv_RT"][0], z["mv_K"], cb, H, W, device=dev)
    ro, rd, near, far = ro[None], rd[None], near[None], far[None]
    sp = ren.prepare_sp_input(batch)
    vol = net.encode_sparse_voxels(sp)
    modes = (0, args.importance)

    def view(importance):
        cfg.render_importance = importance
        with torch.no_grad():
            return ren.get_pixel_value(ro, rd, near, far, vol, sp, batch)

    # the samples each pass lists for the decoder (stats[1] accumulates over the passes of a call)
    listed = {}
    for m in modes:
        ren.stats = torch.zeros(8, dtype=torch.int64, device=dev)
        view(m)
        listed[m] = int(ren.stats[1])
    ren.stats = None
    host = {m: [] for m in modes}
    device = {m: [] for m in modes}
    for it in range(args.views + 2):
        for m in modes:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            e0.record()
            view(m)
            e1.record()
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            if it >= 2:
                host[m].append(1e3 * (t1 - t0))
                device[m].append(e0.elapsed_time(e1))
    cfg.render_importance = 0
    n = int(ro.shape[1])
    c, f = modes
    res = {"view": "%dx%d" % (H, W), "rays": n, "views": args.views, "precision": args.precision,
           "importance": args.importance, "samples_per_ray": [64, 64 + args.importance],
           "coarse_ms": round(float(np.median(host[c])), 3), "coarse_fine_ms": round(float(np.median(host[f])), 3),
           "coarse_device_ms": round(float(np.median(device[c])), 3),
           "coarse_fine_device_ms": round(float(np.median(device[f])), 3),
           "ratio": round(float(np.median(host[f]) / np.median(host[c])), 2),
           "listed_coarse": listed[c], "listed_fine": listed[f] - listed[c],
           "listed_coarse_frac": round(listed[c] / (n * 64), 4),
           "listed_fine_frac": round((listed[f] - listed[c]) / (n * (64 + args.importance)), 4),
           "gpu": torch.cuda.get_device_name(0)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
