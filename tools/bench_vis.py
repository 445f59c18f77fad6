"""Per-view cost of the demo visualize modes, upstream's path against the drop-ins, alternated view by view in one process,
on synth's body seen from a camera 3 m away, at 512 x 512 (ZJU-MoCap at ratio 0.5) and 1080 x 1080 (People-Snapshot's
size).

    python tools/bench_vis.py [--views 24] [--warmup 3] [--sizes 512,1080]

Two modes:
  rotate:     rotate_smpl_cfg, the plain renderer.  (a) upstream: render_utils.image_rays on the host (demo_case.
              upstream_image_rays, upstream's own numpy operations), the rays' H2D copy, the render, then upstream's
              if_nerf_demo visualize body (restated below: .cpu().numpy(), the float64 scatter, BGR, `mkdir -p` through a
              shell, cv2.imwrite of the float64 image * 255).  (b) the drop-ins: the camera to the renderer (rays on the
              device), the render, the Visualizer drop-in's visualize().
  novel_view: novel_view_cfg, the _mmsk renderer with one all-foreground mask view: (a) the camera path of the merged
              dataset drop-in, then upstream's visualize body; (b) the same render, then visualize().
Per mode and size, medians over `--views` views after `--warmup`:
  a_view_ms / b_view_ms   the view from its camera until visualize returns (b: the render and the frame may still be
                          running on the device and the PNG queued; the writer is drained before the next (a) view,
                          outside the timing);
  b_view_device_done_ms   (b) until the device has finished the view (its PNG may still be queued);
  b_view_to_disk_ms       (b) until that view's PNG is on disk (visualize, then flush());
  b_loop_ms               `--views` (b) views back to back, then flush(), over the views: the loop's rate with the writer
                          overlapping the next render;
  a_visualize_ms / b_visualize_ms   the visualize step alone (a: upstream's body after the render has finished, (b):
                          the visualize() call's host time);
  kernel_ms               nb_vis_frame alone (CUDA events around 50 back-to-back launches, per launch).
The synthetic scene supplies its feature volumes, so the sparse-convolution encode is excluded, as in bench_demo.  Checks
that (a) and (b) wrote identical PNG bytes.  One JSON line per mode and size, with the card's name and power limit."""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def upstream_visualize(output, batch, H, W, white_bkgd, img_root_fmt):
    """lib/visualizers/if_nerf_demo.py's visualize (:16-52), with the output root as a format of the frame index."""
    import cv2
    rgb_pred = output['rgb_map'][0].detach().cpu().numpy()
    mask_at_box = batch['mask_at_box'][0].detach().cpu().numpy()
    mask_at_box = mask_at_box.reshape(H, W)
    img_pred = np.zeros((H, W, 3))
    if white_bkgd:
        img_pred = img_pred + 1
    img_pred[mask_at_box] = rgb_pred
    img_pred = img_pred[..., [2, 1, 0]]
    depth_pred = np.zeros((H, W))
    depth_pred[mask_at_box] = output['depth_map'][0].detach().cpu().numpy()
    img_root = img_root_fmt.format(batch['frame_index'].item())
    os.system('mkdir -p {}'.format(img_root))
    index = batch['view_index'].item()
    cv2.imwrite(os.path.join(img_root, '{:04d}.png'.format(index)), img_pred * 255)


def view_camera(size, scene):
    from oracle import synth
    cb = scene["can_bounds"][0].numpy()
    R, T = synth.look_at_camera(0.5 * (cb[0] + cb[1]).astype(np.float64), 3.0, 20.0)
    RT = np.eye(4)
    RT[:3, :3], RT[:3, 3] = R, T[:, 0]
    f = 537.0 * size / 512.0
    K = np.array([[f, 0, size / 2.0], [0, f, size / 2.0], [0, 0, 1.0]])
    return RT, K, cb


def card():
    from tools.bench_eval import card as c
    return c()


def median_ms(ts):
    return round(float(np.median(ts)) * 1e3, 3)


def bench(mode, size, views, warmup, dev, tmp):
    import torch
    from gpu_utils import make_net_and_renderer
    from oracle import synth
    from tools import demo_case as DC
    from neuralbody_b200 import vis_frame
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.networks.make_network import load_source

    scene = synth.make_scene(H=64, W=64, all_hit=False)
    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.raw_noise_std, cfg.chunk = 64, 0.0, False, 0, 0
    cfg.render_precision = "tc_fp16x3"
    net, ren = make_net_and_renderer(scene, dev)
    net.train(False)
    RT, K, cb = view_camera(size, scene)
    base = {k: scene[k].to(dev) for k in ("coord", "out_sh", "bounds", "R", "Th", "latent_index")}
    base["frame_index"] = torch.tensor([0]).to(dev)
    if mode == "novel_view":
        mod = load_source("neuralbody_b200.lib.networks.renderer.if_nerf_renderer_mmsk",
                          os.path.join(ROOT, "neuralbody_b200", "lib", "networks", "renderer", "if_nerf_renderer_mmsk.py"))
        ren = mod.Renderer(net)
        base.update({"msks": torch.ones((1, 1, size, size), dtype=torch.uint8, device=dev),
                     "RT": torch.from_numpy(RT[:3].astype(np.float32))[None, None].to(dev),
                     "Ks": torch.from_numpy(K.astype(np.float32))[None, None].to(dev)})
    cfg.H, cfg.W, cfg.ratio, cfg.exp_name = size, size, 1.0, "bench_vis"
    cam = {"cam_RT": torch.from_numpy(RT)[None], "cam_K": torch.from_numpy(K)[None], "can_bounds": torch.from_numpy(cb)[None]}
    a_root = os.path.join(tmp, "a", mode, "frame_{:04d}")
    os.chdir(os.path.join(tmp, "b"))
    vis = load_source(cfg.visualizer_module, cfg.visualizer_path).Visualizer()

    def path_a(vi):
        return os.path.join(a_root.format(0), "%04d.png" % vi)

    def run_a(vi):
        """-> (view seconds, visualize seconds)"""
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if mode == "rotate":
            ro, rd, nr, fr, m = DC.upstream_image_rays(RT, K, cb, size, size)
            b = dict(base, ray_o=torch.from_numpy(ro)[None].to(dev), ray_d=torch.from_numpy(rd)[None].to(dev),
                     near=torch.from_numpy(nr)[None].to(dev), far=torch.from_numpy(fr)[None].to(dev),
                     mask_at_box=torch.from_numpy(m)[None].to(dev))
        else:
            b = dict(base, meta=cam, **{k: v.to(dev) for k, v in cam.items()})
        b["view_index"] = torch.tensor([vi]).to(dev)
        with torch.no_grad():
            out = ren.render(b)
            torch.cuda.synchronize()         # upstream's .cpu() waits for the render anyway; time its body alone
            t1 = time.perf_counter()
            upstream_visualize(out, b, size, size, False, a_root)
        t2 = time.perf_counter()
        return t2 - t0, t2 - t1

    def run_b(vi, to_disk=False):
        """-> (seconds until visualize() returns, visualize()'s own seconds, seconds until the device is done (or, with
        to_disk, until the PNG is written)); the drop-in's item carries the camera"""
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        b = dict(base, meta=cam, **{k: v.to(dev) for k, v in cam.items()})
        b["view_index"] = torch.tensor([vi]).to(dev)
        with torch.no_grad():
            out = ren.render(b)
            t1 = time.perf_counter()
            vis.visualize(out, b)
        t2 = time.perf_counter()
        torch.cuda.synchronize()
        if to_disk:
            vis.flush()
        return t2 - t0, t2 - t1, time.perf_counter() - t0

    res = {"mode": mode, "size": size, "views": views}
    a_view, a_vis, b_view, b_vis, b_done, b_disk = [], [], [], [], [], []
    for i in range(warmup + views):
        ta = run_a(i)
        tb = run_b(i)
        vis.flush()
        td = run_b(i, to_disk=True)
        if i >= warmup:
            a_view.append(ta[0]); a_vis.append(ta[1])
            b_view.append(tb[0]); b_vis.append(tb[1]); b_done.append(tb[2]); b_disk.append(td[2])
    res.update({"a_view_ms": median_ms(a_view), "b_view_ms": median_ms(b_view), "b_view_device_done_ms": median_ms(b_done),
                "b_view_to_disk_ms": median_ms(b_disk), "a_visualize_ms": median_ms(a_vis),
                "b_visualize_ms": median_ms(b_vis)})
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(views):
        b = dict(base, meta=cam, **{k: v.to(dev) for k, v in cam.items()})
        b["view_index"] = torch.tensor([1000 + i]).to(dev)
        with torch.no_grad():
            vis.visualize(ren.render(b), b)
    vis.flush()
    res["b_loop_ms"] = round((time.perf_counter() - t0) / views * 1e3, 3)
    res["png_identical"] = all(open(path_a(i), "rb").read() ==
                               open(os.path.join(tmp, "b", vis.frame_path(cfg.exp_name, 0, i)), "rb").read()
                               for i in range(warmup + views))
    # the kernel alone
    b = dict(base, meta=cam, **{k: v.to(dev) for k, v in cam.items()})
    with torch.no_grad():
        out = ren.render(b)
    rgb, mask = out["rgb_map"][0].contiguous(), b["mask_at_box"][0].contiguous()
    res["rays"] = int(rgb.shape[0])
    view = vis_frame.ViewFrame(size, size, dev)
    for _ in range(5):
        view.launch(rgb, mask)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(50):
        view.launch(rgb, mask)
    e1.record()
    e1.synchronize()
    res["kernel_ms"] = round(e0.elapsed_time(e1) / 50, 4)
    os.chdir(ROOT)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=24)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sizes", default="512,1080")
    ap.add_argument("--modes", default="rotate,novel_view")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_vis needs a CUDA device")
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    dev = torch.device("cuda:0")
    gpu = card()
    tmp = tempfile.mkdtemp(prefix="bench_vis_")
    try:
        for mode in args.modes.split(","):
            for size in (int(s) for s in args.sizes.split(",")):
                d = os.path.join(tmp, mode, str(size))
                os.makedirs(os.path.join(d, "b"))
                res = bench(mode, size, args.views, args.warmup, dev, d)
                res.update({"card": gpu, "cpus": os.cpu_count()})
                print(json.dumps(res), flush=True)
    finally:
        os.chdir(ROOT)
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
