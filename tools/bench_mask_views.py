"""Measure the demo and mesh datasets' mask steps, upstream's host steps against `dataset_image_steps: 'device'`:
  (a) per item, upstream's host mask steps (binarise, cv2.undistort, cv2.dilate, INTER_NEAREST resize) against the host
      work of a 'device' item (stacking the decoded masks and building the cameras), for the 4-view 1024 x 1024 ZJU-MoCap
      recipe (ratio 0.5) and the 1080 x 1080 People-Snapshot one (ratio 0.5).  Decoding is common to both kinds and left
      out;
  (b) the nb_mask_views call on the GPU for the same recipes, CUDA events over many back-to-back launches;
  (c) two view loops behind a torch DataLoader with the configs' 16 workers (batch size 1, as upstream's visualize
      loader), each item kind in turn in one process (host, device, host, device): the novel-pose loop
      (multi_view_perform_dataset's drop-in -> the _mmsk renderer, a 512 x 512 view) and the mesh frame loop
      (multi_view_mesh_dataset's drop-in -> the mesh renderer with mesh_output 'device').  The data are the full-size
      synthetic body (oracle/synth) and its four 1024 x 1024 training-view masks (distortion 5 coefficients), written as
      PNG and read back with cv2.imread (in place of imageio) by both item kinds.  The loop moves every key but 'meta' to
      the GPU and renders, as upstream's visualize loop does; the visualizers' file writing is left out.  It reports frames/s
      after warm-up, and `alone` lines time the render on one batch of each kind made ahead: the rate the loader has to
      keep up with.
Prints one JSON line per figure, with the GPU's name and power limit and the host's CPU count.

    python -m tools.bench_mask_views [--reps N] [--frames N] [--no-loops]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools import mask_views_case as MC   # noqa: E402

# (name, H0, W0, views' distortions, value set, recipe, ratio)
CASES = (("zju_4x1024", 1024, 1024, ("d5", "d5", "d5", "d5"), "any", "multi_view_perform", 0.5),
         ("snapshot_1080", 1080, 1080, ("d5",), "0255", "monocular_demo", 0.5))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def median_ms(fn, reps):
    fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(t))


def per_item(args, gpu):
    import torch
    from neuralbody_b200 import images
    from neuralbody_b200.lib.datasets import mask_item
    for name, H0, W0, dists, values, recipe, ratio in CASES:
        binarise, dil, _ = MC.RECIPES[recipe]
        msks_u8, Ks, Ds = MC.case(H0, W0, dists, values, 1)
        H, W = MC.out_size(H0, W0, ratio)
        host = median_ms(lambda: [MC.cv2_mask_view(m, K, D, H, W, binarise, dil) for m, K, D in zip(msks_u8, Ks, Ds)],
                         args.reps)
        dev_item = median_ms(lambda: mask_item.mask_fields(list(msks_u8), list(Ks), Ds, H, W, binarise, dil), args.reps)
        keys, meta = mask_item.mask_fields(list(msks_u8), list(Ks), Ds, H, W, binarise, dil)
        x = torch.from_numpy(keys["msks_u8"]).cuda()
        run = lambda: images.mask_views(x, meta["mask_cams"], meta["mask_n_dist"], H, W, binarise, dil)   # noqa: E731
        run()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.launches):
            run()
        e1.record()
        torch.cuda.synchronize()
        print(json.dumps({"case": name, "views": len(dists), "size": [H0, W0], "out": [H, W], "recipe": recipe,
                          "host_mask_steps_ms": round(host, 3), "device_item_host_ms": round(dev_item, 3),
                          "nb_mask_views_ms": round(e0.elapsed_time(e1) / args.launches, 4), "gpu": gpu}), flush=True)


def loop_base(scene, views, root, n_frames, scaled_ratio):
    """A stand-in for upstream's multi-view Dataset over the PNG masks under root/mask_cihp (view v of frame f is file
    f % 2): the attributes the perform and mesh drop-ins read, and get_mask with upstream's host recipe (binarise,
    undistort, 5 x 5 dilation) reading the same files with cv2.imread.  `scaled_ratio`: store Ks scaled by cfg.ratio (the
    demo and perform sets' __init__) or at the masks' size (the mesh set)."""
    import cv2
    Ks, Rs, Ts, _ = views
    nv = len(Ks)
    frame = {k: scene[k][0].numpy() for k in ("coord", "out_sh", "bounds", "Th")}
    Rh = cv2.Rodrigues(scene["R"][0].numpy().astype(np.float64))[0].ravel().astype(np.float32)
    cb = scene["can_bounds"][0].numpy().astype(np.float32)
    D = np.array(MC.DIST["d5"], np.float32)[:, None] * np.float32(0.1)

    class Base:
        def __init__(self):
            self.data_root = root
            self.ims = np.array([["%02d/%06d.jpg" % (v, f % 2) for v in range(nv)] for f in range(n_frames)])
            self.Ks = np.asarray(Ks, np.float32).copy()
            if scaled_ratio:
                self.Ks[:, :2] = self.Ks[:, :2] * np.float32(scaled_ratio)
            self.Ds = np.tile(D, (nv, 1, 1))
            self.Rs, self.Ts = np.asarray(Rs, np.float32), np.asarray(Ts, np.float32)
            self.RT = np.concatenate([self.Rs, self.Ts], axis=2)
            self.K = self.Ks[0]
            self.render_w2c = [self.RT[0]]

        def _host_mask(self, i, v):
            m = cv2.imread(os.path.join(self.data_root, "mask_cihp", self.ims[i][v])[:-4] + ".png", cv2.IMREAD_UNCHANGED)
            m = (m != 0).astype(np.uint8)
            K = self.Ks[v].copy()
            if scaled_ratio:
                K[:2] = K[:2] / scaled_ratio
            m = cv2.undistort(m, K, self.Ds[v])
            return cv2.dilate(m.copy(), np.ones((5, 5), np.uint8))

        def __len__(self):
            return n_frames

        def get_mask(self, i, v=None):
            return self._host_mask(i, v) if v is not None else [self._host_mask(i, u) for u in range(nv)]

        def prepare_input(self, i):
            return frame["coord"], frame["out_sh"], cb, frame["bounds"], Rh, frame["Th"]
    return Base


def loops(args, gpu):
    import cv2
    import torch
    from oracle import mesh_case, synth
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.networks.make_network import load_source
    from neuralbody_b200.lib.datasets.light_stage import multi_view_mesh_dataset, multi_view_perform_dataset
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from gpu_utils import make_net_and_renderer
    dev = torch.device("cuda:0")
    scene = synth.make_scene(**mesh_case.CASES["mesh_full"][0])
    masks = synth.make_mask_views(scene, nv=4, H=1024, W=1024, radius=12)
    views = mesh_case._views(masks)
    net, _ = make_net_and_renderer(scene)
    net.eval()
    rdir = os.path.join(ROOT, "neuralbody_b200", "lib", "networks", "renderer")
    mmsk = load_source("neuralbody_b200.lib.networks.renderer.if_nerf_renderer_mmsk",
                       os.path.join(rdir, "if_nerf_renderer_mmsk.py")).Renderer(net)
    mesh = load_source("neuralbody_b200.lib.networks.renderer.if_mesh_renderer",
                       os.path.join(rdir, "if_mesh_renderer.py")).Renderer(net)
    imread = lambda p: cv2.imread(p, cv2.IMREAD_UNCHANGED)     # noqa: E731
    cfg.H, cfg.W, cfg.ratio, cfg.begin_ith_frame, cfg.chunk = 1024, 1024, 0.5, 0, 0
    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.raw_noise_std = 64, 0.0, False, 0
    cfg.render_precision, cfg.mesh_th, cfg.mesh_output = "tc_fp16x3", 10.0, "device"
    n = args.frames + 4

    def render(ren, batch):
        batch = {k: (v if k == "meta" else v.to(dev)) for k, v in batch.items()}
        with torch.no_grad():
            out = ren.render(batch)
        return out

    with tempfile.TemporaryDirectory() as root:
        for v in range(4):
            os.makedirs(os.path.join(root, "mask_cihp", "%02d" % v))
            for f in range(2):      # part labels over the silhouette, as mask_cihp carries them
                m = masks["msks"][0, v].numpy() * np.uint8(1 + 13 * f)
                cv2.imwrite(os.path.join(root, "mask_cihp", "%02d" % v, "%06d.png" % f), m)
        arms = (("novel_pose_mmsk", multi_view_perform_dataset.make_dataset_class(
                    loop_base(scene, views, root, n, 0.5), cv2=cv2, imread=imread), mmsk),
                ("mesh_frame", multi_view_mesh_dataset.make_dataset_class(
                    loop_base(scene, views, root, n, None), rodrigues=cv2.Rodrigues, imread=imread), mesh))
        for name, cls, ren in arms:
            for mode in ("host", "device"):            # the render alone, on one batch made ahead
                cfg.dataset_image_steps = mode
                one = torch.utils.data.default_collate([cls()[0]])
                for _ in range(3):
                    render(ren, dict(one))
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(args.frames):
                    render(ren, dict(one))
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                print(json.dumps({"loop": name, "alone": mode, "frames": args.frames,
                                  "ms_per_frame": round(dt * 1e3 / args.frames, 2), "gpu": gpu}), flush=True)
            for rep in range(args.loop_reps):
                for mode in ("host", "device"):
                    cfg.dataset_image_steps = mode     # the workers fork with it
                    loader = torch.utils.data.DataLoader(cls(), batch_size=1, shuffle=False, num_workers=args.workers)
                    t0 = None
                    for i, batch in enumerate(loader):
                        if i == 4:
                            torch.cuda.synchronize()
                            t0 = time.perf_counter()
                        render(ren, batch)
                    torch.cuda.synchronize()
                    dt = time.perf_counter() - t0
                    print(json.dumps({"loop": name, "items": mode, "repeat": rep, "workers": args.workers,
                                      "frames": n - 4, "frames_per_s": round((n - 4) / dt, 2),
                                      "ms_per_frame": round(dt * 1e3 / (n - 4), 2), "host_cpus": os.cpu_count(),
                                      "gpu": gpu}), flush=True)
                    del loader
        cfg.dataset_image_steps = "host"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--frames", type=int, default=40, help="timed frames per loop run, after 4 warm-up frames")
    ap.add_argument("--loop-reps", type=int, default=2)
    ap.add_argument("--workers", type=int, default=16)
    ap.add_argument("--no-loops", action="store_true")
    args = ap.parse_args()
    gpu = gpu_info()
    per_item(args, gpu)
    if not args.no_loops:
        loops(args, gpu)


if __name__ == "__main__":
    main()
