"""Host cost of a training item's rays, upstream's against the drop-in's, the GPU sampler's cost, and training steps/s
behind a DataLoader fed with either kind of item.

    python tools/bench_train_data.py [--reps 20] [--steps 40] [--no-loader]

Two seeded synthetic views, written to a temporary directory as PNG with cv2.imwrite and read back with cv2.imread (in
place of imageio): a ZJU-MoCap-313-like one (a 1024 x 1024 view at ratio 0.5 -> 512 x 512, float64 camera) and a
People-Snapshot-like one (1080 x 1080 at ratio 1.0, float32 K).  Per view it prints the medians of
  - upstream: tools.train_rays_case.upstream_sample, upstream's float64 get_rays, np.argwhere and rejection rounds;
  - drop-in: the class map, the empty-list check and the camera the drop-in item computes in its place;
  - the rays.train_rays call (CUDA events around the whole call: camera upload, workspace, the three scans, the list
    scatter, the sampler, the status copy) and the host-to-device copy of the item's image and class map;
with the card's name and power limit.  One JSON line per view.  Then (`item_steps`) per raw view (313-like 1024 x 1024 at
ratio 0.5, Snapshot-like 1080 x 1080 at ratio 1, with distortion) the host ms of decoding, of the rest of a 'host' item
(upstream's undistort, resize, background, class map, camera) and of the rest of a 'device' item, and the nb_item_images
call (CUDA events), with the host CPU count.

Then the loader (`loader_steps`): seeded synthetic data roots of the same two kinds around the synthetic body of
tools/mesh_mono_case (313-like: four 1024 x 1024 views, ratio 0.5, float64 K; Snapshot-like: one 1080 x 1080 view, ratio
1.0, float32 K), PNGs written with cv2.imwrite and read back with cv2.imread in place of imageio.  A map-style dataset runs
upstream's image steps (decode, undistort, INTER_AREA / INTER_NEAREST resize, background) and then either upstream's
sampler on the host (`upstream_sample`, the item carries the rays) or the drop-in's fields (`train_item.train_fields`, the
GPU samples them).  A torch DataLoader at the configs' worker counts (8 for 313, 16 for Snapshot), batch size 1, pinned,
feeds a c3-like step: Renderer.render (64 + 128 samples, training precision), the trainer's mse loss, backward, Adam.
A third item kind, `device` (`dataset_image_steps: 'device'`), stops after decoding and the mask's border and ships the
decoded image and mask; Renderer.render runs nb_item_images on it.  The three loaders alternate in one process (A B C A B
C); each reports steps/s over `--steps` steps after 8 warm-up
steps (one JSON line per view kind, item kind and repeat).  `step_alone` lines time the same step on one item of each kind
made ahead and kept in pinned memory: the rate the loader has to keep up with."""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools import train_rays_case as TC  # noqa: E402
from neuralbody_b200.lib.datasets import train_item  # noqa: E402


def view(kind, d, seed):
    import cv2
    rng = np.random.RandomState(seed)
    H = W = 512 if kind == "313" else 1080
    f = 1.1 * H
    K = np.array([[f, 0, W / 2 + 3.1], [0, f, H / 2 - 2.3], [0, 0, 1.]])
    yy, xx = np.mgrid[0:H, 0:W]
    body = (((xx - W / 2) / (0.18 * W)) ** 2 + ((yy - H / 2) / (0.42 * H)) ** 2) < 1
    msk = body.astype(np.uint8)
    img = (rng.rand(H, W, 3) * 255).astype(np.uint8)
    cv2.imwrite(os.path.join(d, kind + ".png"), img)
    cv2.imwrite(os.path.join(d, kind + "_m.png"), msk * 255)
    img = cv2.imread(os.path.join(d, kind + ".png")).astype(np.float32) / 255.
    msk = (cv2.imread(os.path.join(d, kind + "_m.png"), cv2.IMREAD_GRAYSCALE) != 0).astype(np.uint8)
    if kind == "313":
        msk[(cv2.dilate(msk, np.ones((5, 5), np.uint8)) - cv2.erode(msk, np.ones((5, 5), np.uint8))) == 1] = 100
        K = K.astype(np.float64)
    else:
        K = K.astype(np.float32)
    R, T = np.eye(3), np.array([[0.], [0.], [0.]])
    z = 3.0
    bounds = np.array([[-0.22 * z, -0.45 * z, z - 0.3], [0.22 * z, 0.45 * z, z + 0.3]], np.float32)
    bound = np.zeros((H, W), np.uint8)
    bound[int(0.02 * H):int(0.98 * H), int(0.28 * W):int(0.72 * W)] = 1
    cmap = (train_item.class_map_h36m if kind == "313" else train_item.class_map_snapshot)(msk, bound)
    return img, msk, bound, cmap, K, R, T, bounds


def med(fn, reps):
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t)
    return float(np.median(ts)) * 1e3


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


class SynthTrainData:
    """A training dataset over PNG views: upstream's image steps, then upstream's rays or the drop-in's fields."""

    def __init__(self, paths, K, ratio, h36m, scene_item, mode, n_rand=1024, length=64):
        self.paths, self.K, self.ratio, self.h36m, self.scene_item = paths, K, ratio, h36m, scene_item
        self.mode, self.n_rand, self.length = mode, n_rand, length

    def __len__(self):
        return self.length

    def __getitem__(self, index):
        import cv2
        img_path, msk_path = self.paths[index % len(self.paths)]
        img = cv2.imread(img_path).astype(np.float32) / 255.
        msk = (cv2.imread(msk_path, cv2.IMREAD_GRAYSCALE) != 0).astype(np.uint8)
        if self.h36m:     # multi_view_dataset.get_mask's border
            k = np.ones((5, 5), np.uint8)
            msk[(cv2.dilate(msk.copy(), k) - cv2.erode(msk.copy(), k)) == 1] = 100
        K = self.K.copy()
        D = np.zeros(5)
        img = cv2.undistort(img, K.astype(np.float64), D)
        msk = cv2.undistort(msk, K.astype(np.float64), D)
        H, W = int(img.shape[0] * self.ratio), int(img.shape[1] * self.ratio)
        img = cv2.resize(img, (W, H), interpolation=cv2.INTER_AREA)
        msk = cv2.resize(msk, (W, H), interpolation=cv2.INTER_NEAREST)
        img[msk == 0] = 0
        K[:2] = K[:2] * self.ratio
        ys, xs = np.nonzero(msk)
        bound = np.zeros((H, W), np.uint8)          # stands in for get_bound_2d_mask: the same in both modes
        bound[max(ys.min() - 20, 0):ys.max() + 21, max(xs.min() - 20, 0):xs.max() + 21] = 1
        cmap = (train_item.class_map_h36m if self.h36m else train_item.class_map_snapshot)(msk, bound)
        R, T = np.eye(3), np.zeros((3, 1))
        cb = self.scene_item["can_bounds"]
        ret = {k: v for k, v in self.scene_item.items() if k != "can_bounds"}
        if self.mode == "device":
            return self._device_item(img_path, msk_path)
        if self.mode == "upstream":
            rgb, ray_o, ray_d, near, far = TC.upstream_sample(img, cmap, K, R, T, cb, self.n_rand, 0.5, 0.0)
            ret.update({"rgb": rgb, "ray_o": ray_o, "ray_d": ray_d, "near": near, "far": far,
                        "mask_at_box": np.ones(len(near), bool)})
        else:
            ret.update(train_item.train_fields(img, cmap, K, R, T, cb, self.n_rand, 0.5, 0.0))
        return ret

    def _device_item(self, img_path, msk_path):
        """`dataset_image_steps: 'device'`: decode and the mask's border on the host, the rest on the GPU."""
        import cv2
        img_u8 = cv2.imread(img_path)
        msk = (cv2.imread(msk_path, cv2.IMREAD_GRAYSCALE) != 0).astype(np.uint8)
        if self.h36m:
            k = np.ones((5, 5), np.uint8)
            msk[(cv2.dilate(msk.copy(), k) - cv2.erode(msk.copy(), k)) == 1] = 100
        H, W = int(img_u8.shape[0] * self.ratio), int(img_u8.shape[1] * self.ratio)
        s = img_u8.shape[0] // H
        ys, xs = np.nonzero(msk[::s, ::s])
        bound = np.zeros((H, W), np.uint8)          # stands in for get_bound_2d_mask
        bound[max(ys.min() - 20, 0):ys.max() + 21, max(xs.min() - 20, 0):xs.max() + 21] = 1
        K = self.K.copy()
        Ks = K.copy()
        Ks[:2] = Ks[:2] * self.ratio
        ret = {k: v for k, v in self.scene_item.items() if k != "can_bounds"}
        fields, meta = train_item.device_fields(img_u8, msk, K, np.zeros(5), H, W, True, False, False,
                                                train_item.CLASS_H36M if self.h36m else train_item.CLASS_SNAPSHOT, bound)
        ret.update(fields)
        ret.update(train_item.camera_fields(Ks, np.eye(3), np.zeros((3, 1)), self.scene_item["can_bounds"], self.n_rand,
                                            0.5, 0.0))
        ret["meta"].update(meta)
        return ret


def loader_steps(reps, steps):
    import cv2
    import torch
    from tools import mesh_mono_case as MM
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from gpu_utils import make_net_and_renderer
    from neuralbody_b200.lib.config import cfg
    scene = MM.make_scene(0.3)
    scene_item = {k: scene[k][0].numpy() for k in ("coord", "out_sh", "bounds", "R", "Th", "latent_index")}
    scene_item["can_bounds"] = scene["can_bounds"][0].numpy().astype(np.float32)
    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.raw_noise_std, cfg.chunk = 64, 1.0, False, 0, 0
    cfg.render_importance, cfg.render_train_precision = 128, "tc_tf32x3"
    dev = torch.device("cuda:0")
    net, ren = make_net_and_renderer(scene)
    net.train(True)
    opt = torch.optim.Adam([p for p in net.parameters() if p.requires_grad], lr=5e-4)
    rng = np.random.RandomState(0)
    with tempfile.TemporaryDirectory() as d:
        views = []
        for kind, raw, ratio, nv, workers in (("313", 1024, 0.5, 4, 8), ("snapshot", 1080, 1.0, 1, 16)):
            K = MM.get_camera(MM.camera_pkl(scene, raw, raw))["K"]
            msk = MM.silhouette(scene, K, raw, raw, 2)
            paths = []
            for v in range(nv):
                ip, mp = os.path.join(d, "%s_%d.png" % (kind, v)), os.path.join(d, "%s_%d_m.png" % (kind, v))
                cv2.imwrite(ip, (rng.rand(raw, raw, 3) * 255).astype(np.uint8))
                cv2.imwrite(mp, msk)
                paths.append((ip, mp))
            views.append((kind, paths, K if kind == "313" else K.astype(np.float32), ratio, workers))
        def step(batch):
            batch = {k: (v if k == "meta" else v.to(dev, non_blocking=True)) for k, v in batch.items()}
            ret = ren.render(batch)
            mask = batch["mask_at_box"]
            loss = torch.mean((ret["rgb_map"][mask] - batch["rgb"][mask]) ** 2)
            if "rgb0" in ret:
                loss = loss + torch.mean((ret["rgb0"] - batch["rgb"]) ** 2)
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()

        for kind, paths, K, ratio, workers in views:
            # the step alone, on one pinned item of each kind made ahead: what the loader has to keep up with
            for mode in ("upstream", "dropin", "device"):
                ds = SynthTrainData(paths, K, ratio, kind == "313", scene_item, mode)
                one = torch.utils.data.default_collate([ds[0]])
                one = {k: (v if k == "meta" else v.pin_memory()) for k, v in one.items()}
                for _ in range(5):
                    step(dict(one))
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(steps):
                    step(dict(one))
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                print(json.dumps({"step_alone": kind, "items": mode, "steps": steps, "ms_per_step": round(dt * 1e3 / steps, 2),
                                  "card": card()}), flush=True)
            for rep in range(reps):
                for mode in ("upstream", "dropin", "device"):
                    ds = SynthTrainData(paths, K, ratio, kind == "313", scene_item, mode, length=steps + 8)
                    loader = torch.utils.data.DataLoader(ds, batch_size=1, shuffle=True, num_workers=workers,
                                                         pin_memory=True)
                    t0 = None
                    for i, batch in enumerate(loader):
                        if i == 8:
                            torch.cuda.synchronize()
                            t0 = time.perf_counter()
                        step(batch)
                    torch.cuda.synchronize()
                    dt = time.perf_counter() - t0
                    print(json.dumps({"loader": kind, "items": mode, "repeat": rep, "workers": workers,
                                      "steps": len(ds) - 8, "steps_per_s": round((len(ds) - 8) / dt, 2),
                                      "ms_per_step": round(dt * 1e3 / (len(ds) - 8), 2), "card": card()}), flush=True)
                    del loader


def item_steps(kind, raw, ratio, d, reps, gpu):
    """One raw view's host ms split into decode (cv2.imread of the image and mask) and the rest: upstream's image steps
    with the drop-in's fields ('host' items), or the 'device' item's fields; and the nb_item_images call (CUDA events)."""
    import cv2
    rng = np.random.RandomState(1)
    f = 1.1 * raw
    K = np.array([[f, 0, raw / 2 + 3.1], [0, f, raw / 2 - 2.3], [0, 0, 1.]])
    D = np.array([-0.3, 0.1, 0.001, -0.001, 0.0])
    ip, mp = os.path.join(d, "raw_%s.png" % kind), os.path.join(d, "raw_%s_m.png" % kind)
    yy, xx = np.mgrid[0:raw, 0:raw]
    msk = ((((xx - raw / 2) / (0.18 * raw)) ** 2 + ((yy - raw / 2) / (0.42 * raw)) ** 2) < 1).astype(np.uint8)
    cv2.imwrite(ip, (rng.rand(raw, raw, 3) * 255).astype(np.uint8))
    cv2.imwrite(mp, msk)
    H = W = int(raw * ratio)
    bound = np.ones((H, W), np.uint8)
    h36m = kind == "313"
    cls = train_item.class_map_h36m if h36m else train_item.class_map_snapshot
    Ks = K.copy()
    Ks[:2] *= ratio
    R, T, cb = np.eye(3), np.array([[0.], [0.], [3.]]), np.array([[-1, -1, 2], [1, 1, 4]], np.float32)
    decode = med(lambda: (cv2.imread(ip), cv2.imread(mp, cv2.IMREAD_GRAYSCALE)), reps)
    img_u8, msk_u8 = cv2.imread(ip), cv2.imread(mp, cv2.IMREAD_GRAYSCALE)

    def host():
        img = cv2.undistort(img_u8.astype(np.float32) / 255., K, D)
        m = cv2.undistort(msk_u8, K, D)
        img = cv2.resize(img, (W, H), interpolation=cv2.INTER_AREA)
        m = cv2.resize(m, (W, H), interpolation=cv2.INTER_NEAREST)
        img[m == 0] = 0
        return train_item.train_fields(img, cls(m, bound), Ks, R, T, cb, 1024, 0.5, 0.0)

    def device():
        fields, meta = train_item.device_fields(img_u8, msk_u8, K, D, H, W, True, False, not h36m,
                                                train_item.CLASS_H36M if h36m else train_item.CLASS_SNAPSHOT, bound)
        return fields, meta, train_item.camera_fields(Ks, R, T, cb, 1024, 0.5, 0.0)
    rec = {"item_steps": kind, "raw": raw, "ratio": ratio, "decode_ms": round(decode, 2),
           "host_rest_ms": round(med(host, reps), 2), "device_item_rest_ms": round(med(device, reps), 2),
           "cpus": os.cpu_count(), "card": card()}
    if gpu:
        import torch
        from neuralbody_b200 import images
        dev = torch.device("cuda:0")
        n_dist, cam = images.item_camera(K, D)
        gi = torch.from_numpy(img_u8[None].copy()).to(dev)
        gm = torch.from_numpy(msk_u8[None].copy()).to(dev)
        gb = torch.from_numpy(bound[None].copy()).to(dev)
        rule = images.capi.NB_ITEM_CLASS_H36M if h36m else images.capi.NB_ITEM_CLASS_SNAPSHOT
        call = lambda: images.item_images(gi, gm, cam[None], n_dist, H, W, 1, rule, gb)
        call()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ts = []
        for _ in range(reps):
            e0.record()
            call()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        rec["item_images_call_ms"] = round(float(np.median(ts)), 3)
    return rec


def main():
    import argparse
    import torch
    from neuralbody_b200 import rays
    p = argparse.ArgumentParser()
    p.add_argument("--reps", type=int, default=20)
    p.add_argument("--n-rand", type=int, default=1024)
    p.add_argument("--steps", type=int, default=150)
    p.add_argument("--no-loader", action="store_true")
    a = p.parse_args()
    gpu = torch.cuda.is_available()
    with tempfile.TemporaryDirectory() as d:
        for seed, kind in enumerate(("313", "snapshot")):
            img, msk, bound, cmap, K, R, T, bounds = view(kind, d, seed)
            np.random.seed(0)
            up = med(lambda: TC.upstream_sample(img, cmap, K, R, T, bounds, a.n_rand, 0.5, 0.0), a.reps)
            cm_fn = train_item.class_map_h36m if kind == "313" else train_item.class_map_snapshot
            mine = med(lambda: train_item.train_fields(img, cm_fn(msk, bound), K, R, T, bounds, a.n_rand, 0.5, 0.0), a.reps)
            rec = {"view": kind, "H": img.shape[0], "W": img.shape[1], "n_rand": a.n_rand,
                   "upstream_sampler_ms": round(up, 2), "dropin_host_ms": round(mine, 2), "card": card()}
            if gpu:
                dev = torch.device("cuda:0")
                kk, cam = rays.train_camera(K, R, T, bounds)
                himg = torch.from_numpy(img[None].copy()).pin_memory()
                hcm = torch.from_numpy(cmap[None].copy()).pin_memory()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ts = []
                for _ in range(a.reps):
                    e0.record()
                    gi, gc = himg.to(dev, non_blocking=True), hcm.to(dev, non_blocking=True)
                    e1.record()
                    torch.cuda.synchronize()
                    ts.append(e0.elapsed_time(e1))
                rec["h2d_bytes"] = int(himg.numel() * 4 + hcm.numel())
                rec["h2d_ms"] = round(float(np.median(ts)), 3)
                rays.train_rays(gi, gc, cam[None], kk, a.n_rand, 0.5, 0.0).check()
                ts = []
                for _ in range(a.reps):
                    e0.record()
                    r = rays.train_rays(gi, gc, cam[None], kk, a.n_rand, 0.5, 0.0)
                    e1.record()
                    r.check()
                    ts.append(e0.elapsed_time(e1))
                rec["train_rays_call_ms"] = round(float(np.median(ts)), 3)
            print(json.dumps(rec), flush=True)
        for kind, raw, ratio in (("313", 1024, 0.5), ("snapshot", 1080, 1.0)):
            print(json.dumps(item_steps(kind, raw, ratio, d, a.reps, gpu)), flush=True)
    if gpu and not a.no_loader:
        loader_steps(2, a.steps)


if __name__ == "__main__":
    main()
