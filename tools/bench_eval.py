"""Per-view cost of evaluation, upstream's evaluator path against the drop-in (lib/evaluators/if_nerf.py), on a test-split
view of the synth-313 scene rendered through the test-split path (the item carries the image and camera; Renderer.render
builds the rays, rgb and mask_at_box on the device), at 512 x 512 (ZJU-MoCap 313 at ratio 0.5) and 1080 x 1080
(People-Snapshot's size).

    python tools/bench_eval.py [--views 24] [--warmup 4] [--sizes 512,1080]

Per size, medians over `--views` views after `--warmup`:
  (a) upstream: the rays, rgb and mask copied to the host, then oracle/eval_metrics.evaluate_view with its numpy scatter,
      cv2.boundingRect crop, the two PNGs from the float64 images, and scipy SSIM (skimage 0.14.2's restatement);
  (b) the drop-in's evaluate() wall time, and the time until its two PNGs are on disk (evaluate, then the writer drained);
  (c) nb_eval_image's device time (CUDA events around the launch, back to back);
  (d) render + evaluate per view, both ways (the drop-in's PNGs written while the next view renders; its figure is the
      loop's total, including the last writes, over the views).
One JSON line per size, with the card's name and power limit, and the render alone for context."""
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


def test_view(size, device, seed=0):
    """(scene, batch): the synth-313 body and a size x size test-split item for it, as this package's
    multi_view_dataset drop-in makes one (`img` and the camera under 'meta'), with a random image, collated and moved to
    `device` as upstream's evaluate loop moves it."""
    import torch
    from oracle import synth
    from neuralbody_b200.lib.datasets import train_item
    scene = synth.make_scene(H=64, W=64, all_hit=False)
    cb = scene["can_bounds"][0].numpy()
    center = 0.5 * (cb[0] + cb[1]).astype(np.float64)
    R, T = synth.look_at_camera(center, 3.0, 20.0)
    f = 537.0 * size / 512.0
    K = np.array([[f, 0, size / 2.0], [0, f, size / 2.0], [0, 0, 1.0]])
    rng = np.random.RandomState(seed)
    img = (rng.randint(0, 256, (size, size, 3)).astype(np.float32) / np.float32(255))
    fields = train_item.test_fields(img, K, R, T, cb)
    batch = {k: scene[k].to(device) for k in ("coord", "out_sh", "bounds", "R", "Th", "latent_index")}
    batch["img"] = torch.from_numpy(fields["img"])[None].to(device)
    batch["meta"] = {k: torch.as_tensor(np.asarray(v))[None] for k, v in fields["meta"].items()}
    batch["frame_index"] = torch.tensor([0]).to(device)
    batch["cam_ind"] = torch.tensor([0]).to(device)
    return scene, batch


def card():
    import subprocess
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def median_ms(ts):
    return round(float(np.median(ts)) * 1e3, 3)


def bench_size(size, views, warmup, dev):
    import torch
    from gpu_utils import make_net_and_renderer
    from oracle import eval_metrics as O
    from neuralbody_b200 import metrics
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.networks.make_network import load_source

    scene, batch = test_view(size, dev)
    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.raw_noise_std, cfg.chunk = 64, 0.0, False, 0, 0
    cfg.render_precision = "tc_fp16x3"
    _, ren = make_net_and_renderer(scene, dev)
    tmp = tempfile.mkdtemp(prefix="bench_eval_")
    cfg.H, cfg.W, cfg.ratio, cfg.eval_whole_img, cfg.result_dir = size, size, 1.0, False, tmp
    ev = load_source(cfg.evaluator_module, cfg.evaluator_path).Evaluator()
    png_dir = os.path.join(tmp, "upstream")
    os.makedirs(png_dir)

    def render():
        with torch.no_grad():
            return ren.render(batch)

    def upstream(out):
        pred = out["rgb_map"][0].detach().cpu().numpy()
        gt = batch["rgb"][0].detach().cpu().numpy()
        mask = batch["mask_at_box"][0].detach().cpu().numpy()
        return O.evaluate_view(pred, gt, mask, size, size, png_dir=png_dir)

    out = render()
    torch.cuda.synchronize()
    n_rays = int(out["rgb_map"].shape[1])
    res = {"size": size, "rays": n_rays, "views": views}

    def timed(fn, sync=False):
        ts = []
        for i in range(warmup + views):
            t = time.perf_counter()
            fn()
            if sync:
                torch.cuda.synchronize()
            if i >= warmup:
                ts.append(time.perf_counter() - t)
        return ts

    res["render_ms"] = median_ms(timed(render, sync=True))
    ref = upstream(out)
    res["box"] = list(ref["box"])
    res["a_upstream_eval_ms"] = median_ms(timed(lambda: upstream(out)))
    res["b_dropin_evaluate_ms"] = median_ms(timed(lambda: ev.evaluate(out, batch)))
    ev._writer.join()

    def to_disk():
        ev.evaluate(out, batch)
        ev._writer.join()
    res["b_dropin_pngs_on_disk_ms"] = median_ms(timed(to_disk))
    got = ev.ssim[-1]
    res["ssim_upstream"], res["ssim_dropin"] = float(ref["ssim"]), float(got)

    # (c) the kernels alone, back to back on the stream
    pred, gt, mask = out["rgb_map"][0].contiguous(), batch["rgb"][0].contiguous(), batch["mask_at_box"][0].contiguous()
    view = metrics.ViewEval(size, size, dev)
    for _ in range(warmup):
        view.launch(pred, gt, mask)
    ks = []
    for _ in range(views):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        view.launch(pred, gt, mask)
        b.record()
        b.synchronize()
        ks.append(a.elapsed_time(b) / 1e3)
    res["c_kernels_ms"] = median_ms(ks)

    # (d) render + evaluate per view
    res["d_render_upstream_eval_ms"] = median_ms(timed(lambda: upstream(render())))
    for _ in range(warmup):
        ev.evaluate(render(), batch)
    ev._writer.join()
    t = time.perf_counter()
    per = []
    for _ in range(views):
        t1 = time.perf_counter()
        ev.evaluate(render(), batch)
        per.append(time.perf_counter() - t1)
    ev._writer.join()
    res["d_render_dropin_eval_ms"] = round((time.perf_counter() - t) / views * 1e3, 3)
    res["d_render_dropin_eval_median_view_ms"] = median_ms(per)
    ev.mse, ev.psnr, ev.ssim = [], [], []
    shutil.rmtree(tmp, ignore_errors=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=24)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--sizes", default="512,1080")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval needs a CUDA device")
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    dev = torch.device("cuda:0")
    gpu = card()
    for size in (int(s) for s in args.sizes.split(",")):
        res = bench_size(size, args.views, args.warmup, dev)
        res.update({"card": gpu, "cpus": os.cpu_count()})
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
