"""Per-view cost of the demo datasets' rays: upstream's data path (image_rays on the host with upstream's own numpy operations,
demo_case.upstream_image_rays, + the mask views' undistort / dilate / resize, the H2D copy of the rays, the render) against the camera path (the mask views as before, the camera to
the renderer, nb_image_rays on the device, the same render), alternated view by view in one process; medians.

    python -m tools.bench_demo [--views 20] [--precision tc_fp16x3]

The view is a full-size gen_path orbit view (tests/golden/demo_orbit_s512.npz, float64 camera) over synth's full-size
body; the four mask views are synthetic 1024 x 1024 silhouettes (decode not included).  Also reports the ray kernel alone
(CUDA events)."""
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


def host_masks(msks, K, D, H, W):
    import cv2
    out = []
    for m, k, d in zip(msks, K, D):
        m = cv2.undistort(m, k, d)
        m = cv2.dilate(m.copy(), np.ones((5, 5), np.uint8))
        out.append(cv2.resize(m, (W, H), interpolation=cv2.INTER_NEAREST))
    return np.array(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=20)
    ap.add_argument("--precision", default="tc_fp16x3")
    args = ap.parse_args()
    from neuralbody_b200 import rays
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.networks.make_network import load_source
    from tools import mesh_mono_case as MM
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from gpu_utils import make_net_and_renderer
    z = np.load(DC.ORBIT)
    K = z["mv_K"]
    H, W = (int(v) for v in z["mv_HW"])
    scene = MM.make_scene(1.0)
    # the orbit's cameras look at the origin, where synth's full-size body sits: its can_bounds is the view's box
    cb = scene["can_bounds"][0].numpy()
    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.raw_noise_std = 64, 0.0, False, 0
    cfg.render_precision, cfg.chunk = args.precision, 0
    net, _ = make_net_and_renderer(scene)
    net.train(False)
    mod = load_source("neuralbody_b200.lib.networks.renderer.if_nerf_renderer_mmsk",
                      os.path.join(ROOT, "neuralbody_b200", "lib", "networks", "renderer", "if_nerf_renderer_mmsk.py"))
    ren = mod.Renderer(net)
    cfg.H, cfg.W, cfg.ratio = 2 * H, 2 * W, 0.5
    rng = np.random.RandomState(0)
    raw = [(rng.rand(1024, 1024) > 0.7).astype(np.uint8) for _ in range(4)]
    Km = [np.array([[1100., 0, 512], [0, 1100., 512], [0, 0, 1]], np.float32)] * 4
    Dm = [DC.DIST.astype(np.float32)] * 4
    RTm = torch.from_numpy(np.stack([np.eye(4)[:3]] * 4).astype(np.float32))[None].cuda()
    Kms = torch.from_numpy(np.stack(Km) * np.array([[.5], [.5], [1]], np.float32))[None].cuda()
    dev = "cuda:0"
    base = {k: scene[k].to(dev) for k in ("coord", "out_sh", "bounds", "R", "Th", "latent_index")}
    t_up, t_cam, t_kernel, n_rays = [], [], [], []
    for it in range(args.views + 2):
        RT = z["mv_RT"][it % len(z["mv_RT"])]
        # upstream: host rays + masks, H2D, render
        torch.cuda.synchronize(); t0 = time.perf_counter()
        msks = host_masks(raw, Km, Dm, H, W)
        ro, rd, nr, fr, m = DC.upstream_image_rays(RT, K, cb, H, W)     # upstream's own numpy operations
        b = dict(base, msks=torch.from_numpy(msks)[None].to(dev), RT=RTm, Ks=Kms,
                 ray_o=torch.from_numpy(ro)[None].to(dev), ray_d=torch.from_numpy(rd)[None].to(dev),
                 near=torch.from_numpy(nr)[None].to(dev), far=torch.from_numpy(fr)[None].to(dev))
        with torch.no_grad():
            out_a = ren.render(b)
        torch.cuda.synchronize(); t1 = time.perf_counter()
        # camera path: host masks, the camera (on the device, and its host copy in 'meta' as the drop-ins and upstream's
        # visualize loop leave it), device rays, render
        msks = host_masks(raw, Km, Dm, H, W)
        cam = {"cam_RT": torch.from_numpy(RT)[None], "cam_K": torch.from_numpy(K)[None], "can_bounds": torch.from_numpy(cb)[None]}
        b = dict(base, msks=torch.from_numpy(msks)[None].to(dev), RT=RTm, Ks=Kms, meta=cam,
                 **{k: v.to(dev) for k, v in cam.items()})
        with torch.no_grad():
            out_b = ren.render(b)
        torch.cuda.synchronize(); t2 = time.perf_counter()
        # the kernel alone
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rays.camera_image_rays(RT, K, cb, H, W)
        e1.record(); torch.cuda.synchronize()
        assert all(torch.equal(out_a[k].view(torch.int32), out_b[k].view(torch.int32)) for k in out_a)   # bits: disp_map has NaN
        if it >= 2:
            t_up.append(t1 - t0); t_cam.append(t2 - t1); t_kernel.append(e0.elapsed_time(e1)); n_rays.append(len(ro))
    print(json.dumps({"view": "%dx%d" % (H, W), "views": args.views, "rays_median": int(np.median(n_rays)),
                      "upstream_ms": round(1e3 * float(np.median(t_up)), 2), "camera_ms": round(1e3 * float(np.median(t_cam)), 2),
                      "image_rays_call_ms": round(float(np.median(t_kernel)), 3), "host_cpus": os.cpu_count(),
                      "gpu": torch.cuda.get_device_name(0)}))


if __name__ == "__main__":
    main()
