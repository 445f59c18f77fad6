"""The evaluator's per-view cases (TEST INFRASTRUCTURE ONLY) and the generator of their golden.

`case(name)` rebuilds a seeded view from integers alone (so every machine rebuilds the same float32 bits): colours k / 255
on ramps with a perturbed prediction and a block of random values, and a mask of the case's shape.  `run_reference`
runs the UNMODIFIED reference evaluator (lib/evaluators/if_nerf.py) through oracle/ref_harness.py, with
skimage.measure.compare_ssim stubbed by oracle/eval_metrics.compare_ssim and termcolor stubbed, and returns its
metrics.npy and PNG bytes.

    python -m tools.eval_case

writes, overwriting it, tests/golden/eval_metrics.npz: per case the reference's mse, psnr, ssim, the crop box and the
decoded uint8 comparison images, and a checksum of the rebuilt inputs."""
import hashlib
import os
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden", "eval_metrics.npz")
# name: (H, W, white_bkgd, eval_whole_img, mask kind, seed)
CASES = {
    "small": (40, 48, 0, 0, "ellipse", 0),
    "zju512": (512, 512, 0, 0, "ellipse", 1),
    "snapshot1080": (1080, 1080, 0, 0, "tall", 2),
    "white": (96, 128, 1, 0, "ellipse", 3),
    "whole": (96, 128, 0, 1, "ellipse", 4),
    "border": (64, 80, 0, 0, "border", 5),
    "holes": (80, 96, 1, 0, "holes", 6),
    "crop7": (50, 60, 0, 0, "bar7", 7),
}


def mask_of(kind, H, W):
    yy, xx = np.mgrid[0:H, 0:W]
    if kind == "ellipse":       # ~ a ZJU-MoCap body's box-hit pixels
        return ((xx - W * 0.47) / (0.21 * W)) ** 2 + ((yy - H * 0.52) / (0.41 * H)) ** 2 < 1
    if kind == "tall":          # People-Snapshot-like: a standing body
        return ((xx - W * 0.5) / (0.2 * W)) ** 2 + ((yy - H * 0.5) / (0.46 * H)) ** 2 < 1
    if kind == "border":        # touching the top, left and right edges
        return (yy < H * 0.6) & ((xx < W * 0.3) | (xx > W * 0.8) | (yy < 5))
    if kind == "holes":         # two components, the larger one with holes
        a = ((xx - W * 0.35) / (0.25 * W)) ** 2 + ((yy - H * 0.5) / (0.4 * H)) ** 2 < 1
        holes = ((xx // 5) % 3 == 0) & ((yy // 7) % 2 == 0)
        b = (np.abs(xx - W * 0.82) < 6) & (np.abs(yy - H * 0.2) < 9)
        return (a & ~holes) | b
    if kind == "bar7":          # a crop exactly 7 pixels wide
        return (xx >= 20) & (xx < 27) & (yy >= 10) & (yy < 40)
    raise ValueError(kind)


def case(name):
    """-> rgb_pred, rgb_gt (n,3) float32, mask (H*W) bool, and the case's (H, W, white_bkgd, eval_whole_img)."""
    H, W, white, whole, kind, seed = CASES[name]
    yy, xx = np.mgrid[0:H, 0:W].astype(np.int64)
    c = np.arange(3, dtype=np.int64)
    k_gt = (3 * xx[..., None] + 5 * yy[..., None] + 40 * c + 17 * seed) % 256
    k_pred = np.clip(k_gt + (xx[..., None] * yy[..., None] + 7 * c) % 17 - 8, 0, 255)
    gt = (k_gt.astype(np.float32) / np.float32(255))
    pred = (k_pred.astype(np.float32) / np.float32(255))
    rng = np.random.RandomState(seed)
    bh, bw = min(24, H // 3), min(24, W // 3)
    y0, x0 = H // 2 - bh // 2, W // 2 - bw // 2
    pred[y0:y0 + bh, x0:x0 + bw] = rng.rand(bh, bw, 3).astype(np.float32)
    mask = mask_of(kind, H, W)
    return pred[mask], gt[mask], mask.reshape(-1), (H, W, white, whole)


def checksum(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def random_view(H, W, seed, special=False):
    """A random-colour view with an ellipse mask (the oracle's random cases); `special` puts the values cv2 saturates or
    rounds on a tie (0.5 -> 127.5, 1.5, -0.1, 1e10, inf, NaN) into the prediction's first rays."""
    rng = np.random.RandomState(seed)
    cy, cx = rng.uniform(0.3, 0.7) * H, rng.uniform(0.3, 0.7) * W
    yy, xx = np.mgrid[0:H, 0:W]
    mask = ((xx - cx) / (rng.uniform(0.15, 0.4) * W)) ** 2 + ((yy - cy) / (rng.uniform(0.2, 0.45) * H)) ** 2 < 1
    n = int(mask.sum())
    pred = rng.rand(n, 3).astype(np.float32)
    gt = np.clip(pred + rng.normal(0, 0.05, (n, 3)), 0, 1).astype(np.float32)
    if special:
        vals = np.array([0.5, 1.5, -0.1, 1e10, np.inf, -np.inf, np.nan, 1.0, 0.0], np.float32)
        pred[:len(vals), 0] = vals
    return pred, gt, mask.reshape(-1)


# ----------------------------------------------------------------------------- the unmodified reference evaluator
def reference_evaluator():
    """The reference's lib/evaluators/if_nerf.py module and its cfg, loaded through oracle/ref_harness.py with
    skimage.measure.compare_ssim = oracle.eval_metrics.compare_ssim and a pass-through termcolor."""
    from oracle import ref_harness, eval_metrics
    cfg = ref_harness.load_reference()[0]
    if "skimage.measure" not in sys.modules:
        sk, skm = types.ModuleType("skimage"), types.ModuleType("skimage.measure")
        skm.compare_ssim = eval_metrics.compare_ssim
        sk.measure = skm
        sys.modules["skimage"], sys.modules["skimage.measure"] = sk, skm
    if "termcolor" not in sys.modules:
        tc = types.ModuleType("termcolor")
        tc.colored = lambda text, *a, **k: text
        sys.modules["termcolor"] = tc
    if ref_harness.REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, ref_harness.REFERENCE_ROOT)
    import importlib
    mod = importlib.import_module("lib.evaluators.if_nerf")
    return mod, cfg


def run_reference(name, frame_index=3, view_index=11):
    """The reference evaluator on case `name` -> dict: mse, psnr, ssim (its metrics.npy entries) and the bytes of its two
    PNG files."""
    mod, cfg = reference_evaluator()
    pred, gt, mask, (H, W, white, whole) = case(name)
    return run_reference_view(mod, cfg, pred, gt, mask, H, W, white, whole, frame_index, view_index)


def run_reference_view(mod, cfg, pred, gt, mask, H, W, white, whole, frame_index=3, view_index=11):
    import torch
    with tempfile.TemporaryDirectory() as d:
        cfg.H, cfg.W, cfg.ratio = H, W, 1.0
        cfg.white_bkgd, cfg.eval_whole_img, cfg.result_dir = bool(white), bool(whole), d
        ev = mod.Evaluator()
        batch = {"rgb": torch.from_numpy(gt)[None], "mask_at_box": torch.from_numpy(mask)[None],
                 "frame_index": torch.tensor([frame_index]), "cam_ind": torch.tensor([view_index])}
        ev.evaluate({"rgb_map": torch.from_numpy(pred)[None]}, batch)
        ev.summarize()
        m = np.load(os.path.join(d, "metrics.npy"), allow_pickle=True).item()
        png = os.path.join(d, "comparison", "frame%04d_view%04d" % (frame_index, view_index))
        out = {k: m[k][0] for k in ("mse", "psnr", "ssim")}
        out["png_pred"] = open(png + ".png", "rb").read()
        out["png_gt"] = open(png + "_gt.png", "rb").read()
    return out


def load_golden():
    z = np.load(GOLDEN)
    return {name: {k: z[name + "_" + k] for k in ("mse", "psnr", "ssim", "box", "crop_pred", "crop_gt", "sha256")}
            for name in CASES}


def main():
    import cv2
    arrays = {}
    for name in CASES:
        pred, gt, mask, _ = case(name)
        ref = run_reference(name)
        H, W, white, whole = CASES[name][:4]
        box = (0, 0, W, H) if whole else tuple(int(v) for v in cv2.boundingRect(mask.reshape(H, W).astype(np.uint8)))
        crops = [cv2.imdecode(np.frombuffer(ref[k], np.uint8), cv2.IMREAD_UNCHANGED) for k in ("png_pred", "png_gt")]
        for k, v in (("mse", ref["mse"]), ("psnr", ref["psnr"]), ("ssim", ref["ssim"]), ("box", np.array(box, np.int32)),
                     ("crop_pred", crops[0]), ("crop_gt", crops[1]),
                     ("sha256", np.frombuffer(checksum(pred, gt, mask).encode(), np.uint8))):
            arrays[name + "_" + k] = np.asarray(v)
        print(name, box, ref["mse"], ref["psnr"], ref["ssim"])
    np.savez_compressed(GOLDEN, **arrays)
    print("wrote", GOLDEN, os.path.getsize(GOLDEN), "bytes")


if __name__ == "__main__":
    main()
